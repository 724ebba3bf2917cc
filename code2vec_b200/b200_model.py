"""`Code2VecModel` for `--framework b200`: the third backend behind Code2VecModelBase.

Where the reference's TensorFlow backend (tensorflow_model.py:18-447) builds a graph and calls
`sess.run`, this class feeds host batches from the reader to the C-ABI engine:
    train()    : c2v_train_batch_host per batch      == sess.run([optimizer, train_loss])   (:80)
    evaluate() : c2v_predict_batch_host per batch    == sess.run([top_words, top_values, ...]) (:157-161)
    predict()  : c2v_predict_batch_host, batch of 1, normalised scores + attention           (:331-335)
Host-side bookkeeping (logging cadence, save/evaluate cadence, log.txt, .vectors, metrics) follows
the reference method by method; the citations are on each method.
Under torch.distributed.run with WORLD_SIZE = 2, 4 or 8, train() and evaluate() run the fully sharded schedule: every
rank takes its slice of each global batch, rank 0 logs and writes the files, and the checkpoint is written and read by
all ranks in the one-GPU format (multi_rank.py, DESIGN.md §6c).
"""
from __future__ import annotations

import contextlib
import json
import os
import struct
import time
from collections import Counter
from functools import partial
from typing import Dict, Iterable, List, Optional

import numpy as np

from .common import common
from .config import Config
from .engine import (PARAM_NAMES, EngineDims, PathAttentionEngine, cols_to_rows, crc32c_combine, crc32c_rows,
                     rows_to_cols, tensor_crc32c)
from .keras_ckpt import keras_entries, keras_layout, latest_checkpoint, record_checkpoint, write_keras_index
from .model_base import Code2VecModelBase, ModelEvaluationResults, ModelPredictionResults
from .path_context_reader import EstimatorAction, ModelInputTensorsFormer, PathContextReader, ReaderInputTensors
from .multi_rank import (CKPT_MAGIC, CKPT_SUFFIX, batch_split, check_checkpoint_dims, check_multi_rank_run,
                         checkpoint_header, create_checkpoint_file, read_checkpoint_header, read_checkpoint_part,
                         read_entries_part, run_world, write_checkpoint, write_checkpoint_part)
from .tf_bundle import INDEX_SUFFIX, bundle_entries, bundle_layout, crc_view, data_file, save_format_flag, write_index
from .tf_bundle import crc32c as host_crc32c
from . import device_reader as _device_reader_mod
from .device_reader import device_eval_flag, device_reader_flag, evaluation_route_line, sharded_reader_flag
from .device_predict import device_predict_flag
from .text_export import DeviceTextWriter, device_text_flag
from .trainer import ADAM_DEFAULTS, Trainer, make_fully_sharded_engine
from .vocabularies import VocabType


def _barrier():
    import torch.distributed as dist
    dist.barrier()

def _prefetch(iterable, depth: int = 8):
    """Runs `iterable` (the reader) in a background thread, `depth` batches ahead: the native
    tensoriser and the C-ABI train call both release the GIL, so parsing the next batches overlaps
    the GPU step -- the role tf.data's prefetch(40) plays in the reference (path_context_reader.py:150)."""
    import queue
    import threading
    q: "queue.Queue" = queue.Queue(maxsize=depth)
    done = object()
    stop = threading.Event()

    def put(item) -> bool:
        while not stop.is_set():
            try:
                q.put(item, timeout=0.1)
                return True
            except queue.Full:
                continue
        return False

    def run():
        try:
            for item in iterable:
                if not put(item):
                    return                    # the consumer went away (endless readers end here)
            put(done)
        except BaseException as exc:          # surface reader errors in the consumer
            put(exc)

    threading.Thread(target=run, daemon=True).start()
    try:
        while True:
            item = q.get()
            if item is done:
                return
            if isinstance(item, BaseException):
                raise item
            yield item
    finally:
        stop.set()


def _with_next(iterable):
    """(item, following item or None) pairs: the one-batch lookahead behind the engine's next-batch hint."""
    it = iter(iterable)
    try:
        cur = next(it)
    except StopIteration:
        return
    for nxt in it:
        yield cur, nxt
        cur = nxt
    yield cur, None


DEFAULT_DETERMINISTIC_SEED = 1       # the seed of a C2V_DETERMINISTIC=1 run that names none


def run_determinism(environ, now=time.time):
    """(deterministic, seed) of a training run from its environment.  C2V_DETERMINISTIC=1 sets the engine option
    "deterministic" (a step's results depend only on its inputs, seeds and options); C2V_SEED=<int >= 0> fixes the dropout
    seed and the training reader's shuffle seed.  Without C2V_SEED the seed is DEFAULT_DETERMINISTIC_SEED in a
    deterministic run and derived from the clock otherwise; it is logged either way, so any run can be replayed."""
    flag = environ.get("C2V_DETERMINISTIC", "0") or "0"
    if flag not in ("0", "1"):
        raise ValueError("C2V_DETERMINISTIC must be 0 or 1, got %r" % flag)
    deterministic = flag == "1"
    raw = environ.get("C2V_SEED", "")
    if raw:
        try:
            seed = int(raw)
        except ValueError:
            raise ValueError("C2V_SEED must be a non-negative integer, got %r" % raw) from None
        if seed < 0:
            raise ValueError("C2V_SEED must be a non-negative integer, got %r" % raw)
    else:
        seed = DEFAULT_DETERMINISTIC_SEED if deterministic else int(now()) & 0x7FFFFFFF
    return deterministic, seed


MAX_NUM_SAMPLED = 1024              # the sampled-softmax head's limit (c2v_sampled_train_step)


def num_sampled_flag(environ) -> int:
    """C2V_NUM_SAMPLED=<S>: train() runs the sampled softmax with S unique log-uniform negatives per step, drawn on the GPU
    (DESIGN.md §6j); 0 (the default) runs the full softmax.  ValueError for anything but a non-negative integer."""
    raw = environ.get("C2V_NUM_SAMPLED", "0") or "0"
    try:
        value = int(raw, 10)
    except ValueError:
        raise ValueError("C2V_NUM_SAMPLED must be a non-negative integer, got %r" % raw) from None
    if value < 0 or raw.strip() != raw:
        raise ValueError("C2V_NUM_SAMPLED must be a non-negative integer, got %r" % raw)
    return value


def check_num_sampled(num_sampled: int, target_vocab: int) -> None:
    """ValueError unless 1 <= num_sampled <= min(1024, floor(target_vocab / 2)): the unique sampler needs at most half of the
    target words, which keeps the expected number of draws per step small."""
    limit = min(MAX_NUM_SAMPLED, target_vocab // 2)
    if not 1 <= num_sampled <= limit:
        raise ValueError("C2V_NUM_SAMPLED=%d is outside [1, %d]: the sampled softmax draws at most min(1024, half of the %d "
                         "target words) negatives; lower it, or set 0 for the full softmax" % (num_sampled, limit, target_vocab))


def sharded_sampled_flag(environ) -> bool:
    """C2V_SHARDED_SAMPLED=1 (with C2V_NUM_SAMPLED=<S>): train() runs the sampled softmax on 2, 4 or 8 GPUs too, on the
    fully sharded schedule (DESIGN.md §6j, "Several GPUs").  0 (the default) keeps the one-GPU-only refusal.  ValueError
    for anything but 0 or 1."""
    flag = environ.get("C2V_SHARDED_SAMPLED", "0") or "0"
    if flag not in ("0", "1"):
        raise ValueError("C2V_SHARDED_SAMPLED must be 0 or 1, got %r" % flag)
    return flag == "1"


def extend_vocab_flag(environ) -> bool:
    """C2V_EXTEND_VOCAB=1: a run that loads (--load) and trains (--data) extends the loaded vocabularies by the dataset's
    words and continues from the loaded model at the merged sizes (DESIGN.md §6m).  "" and "0" (the default) are off.
    ValueError for anything but 0 or 1."""
    flag = environ.get("C2V_EXTEND_VOCAB", "0") or "0"
    if flag not in ("0", "1"):
        raise ValueError("C2V_EXTEND_VOCAB must be 0 or 1, got %r" % flag)
    return flag == "1"


def extend_vocab_run(config, extend: bool, log) -> bool:
    """Whether this run extends its loaded vocabularies (extend: the value of C2V_EXTEND_VOCAB).  A run that does not
    train or does not load logs that the switch has no effect.  ValueError, before anything is read or written, when
    --save puts dictionaries.bin in the --load directory: it would replace the file the loaded checkpoints need."""
    if not extend:
        return False
    if not config.is_training:
        log("C2V_EXTEND_VOCAB=1 has no effect: this run does not train (no --data)")
        return False
    if not config.is_loading:
        log("C2V_EXTEND_VOCAB=1 has no effect: this run does not load a model (no --load), and a model trained from "
            "scratch already takes the dataset's vocabulary")
        return False
    if config.is_saving:
        where = lambda p: os.path.realpath(os.path.dirname(os.path.abspath(Config.get_vocabularies_path_from_model_path(p))))
        folder = where(config.MODEL_LOAD_PATH)
        if where(config.MODEL_SAVE_PATH) == folder:
            raise ValueError("C2V_EXTEND_VOCAB=1: --save writes the extended vocabularies to `%s`, the directory of --load, "
                             "and its dictionaries.bin would no longer fit the loaded checkpoints; save to another "
                             "directory" % os.path.join(folder, "dictionaries.bin"))
    return True


def _lead(t, shape):
    """The leading rows of the engine tensor t that a stored tensor of `shape` fills: all of t unless C2V_EXTEND_VOCAB=1
    grew its table."""
    return t[:int(shape[0])] if len(shape) == 2 else t


class _PinnedStaging:
    """Two page-locked buffers between files and device tensors, as DeviceTextWriter has (DESIGN.md §6f): the host
    fills or drains one while the other's copy runs on the current stream."""
    CHUNK_BYTES = 64 << 20

    def __init__(self, dev, chunk_bytes: int = CHUNK_BYTES):
        import torch
        self.torch = torch
        self.dev = torch.device(dev)
        self.chunk = int(chunk_bytes)
        self.buf = [torch.empty(self.chunk, dtype=torch.uint8, pin_memory=True) for _ in range(2)]
        self.events = [None, None]
        self.slot = 0

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        for ev in self.events:
            if ev is not None:
                ev.synchronize()
        self.buf = self.events = None

    def _take(self) -> int:
        s = self.slot
        self.slot ^= 1
        if self.events[s] is not None:
            self.events[s].synchronize()
        return s

    def _mark(self, s: int):
        ev = self.torch.cuda.Event()
        ev.record(self.torch.cuda.current_stream(self.dev))
        self.events[s] = ev

    def upload(self, path: str, offset: int, nbytes: int, t):
        """Bytes [offset, offset + nbytes) of the file into the contiguous device tensor t."""
        dst = t.view(-1).view(self.torch.uint8)
        with open(path, "rb") as f:
            f.seek(offset)
            for o in range(0, nbytes, self.chunk):
                n = min(self.chunk, nbytes - o)
                s = self._take()
                if f.readinto(memoryview(self.buf[s].numpy())[:n]) != n:
                    raise ValueError("`%s` ends inside the tensor at offset %d" % (path, offset))
                dst[o:o + n].copy_(self.buf[s][:n], non_blocking=True)
                self._mark(s)

    def download(self, t, f):
        """The bytes of the contiguous device tensor t appended to the binary file f."""
        src = t.reshape(-1).view(self.torch.uint8)
        pending = None
        for o in range(0, src.numel(), self.chunk):
            n = min(self.chunk, src.numel() - o)
            s = self._take()
            self.buf[s][:n].copy_(src[o:o + n], non_blocking=True)
            self._mark(s)
            if pending is not None:
                self._write(f, *pending)
            pending = (s, n)
        if pending is not None:
            self._write(f, *pending)

    def _write(self, f, s: int, n: int):
        self.events[s].synchronize()
        f.write(memoryview(self.buf[s].numpy())[:n])


_CKPT_MAGIC = CKPT_MAGIC
_CKPT_SUFFIX = CKPT_SUFFIX


class Code2VecModel(Code2VecModelBase):
    _ADAM: Optional[dict] = None      # None = tf.compat.v1.train.AdamOptimizer() defaults (tensorflow_model.py:232)
    _INIT_SCHEME = "tensorflow"       # engine.init_params's initialisers of a model built from scratch
    _extend_vocab = False             # C2V_EXTEND_VOCAB=1 applies to this run (extend_vocab_run)

    def __init__(self, config: Config):
        self.engine: Optional[PathAttentionEngine] = None
        self.trainer: Optional[Trainer] = None
        self.eval_reader = None
        self.predict_reader = None
        # the reference's TF variable names, kept for checkpoint metadata (tensorflow_model.py:32-36)
        self.vocab_type_to_tf_variable_name_mapping: Dict[VocabType, str] = {
            VocabType.Token: "WORDS_VOCAB", VocabType.Target: "TARGET_WORDS_VOCAB", VocabType.Path: "PATHS_VOCAB"}
        self._param_of_vocab = {VocabType.Token: "tok", VocabType.Target: "tgt", VocabType.Path: "path"}
        # WORLD_SIZE > 1 (torch.distributed.run): one rank per GPU on the fully sharded schedule (DESIGN.md §6c)
        self.world, self.local_rank = run_world(os.environ)
        self.rank = 0
        self._own_group = False
        # C2V_SAVE_FORMAT=tf: save() and --release write TensorFlow V2 checkpoints (tf_bundle.py, DESIGN.md §6k);
        # C2V_SAVE_FORMAT=keras: the reference Keras backend's checkpoints (keras_ckpt.py, DESIGN.md §6l)
        self._save_format = save_format_flag(os.environ)
        check_multi_rank_run(config, self.world, self._save_format)
        # C2V_NUM_SAMPLED=<S>: train() runs the sampled softmax with S negatives drawn on the GPU (DESIGN.md §6j)
        self._num_sampled = num_sampled_flag(os.environ)
        # C2V_SHARDED_SAMPLED=1: the sampled softmax on several GPUs too, rows fetched from their owners (§6j)
        self._sharded_sampled = sharded_sampled_flag(os.environ)
        if self._sharded_sampled and not self._num_sampled:
            raise ValueError("C2V_SHARDED_SAMPLED=1 trains the sampled softmax on several GPUs: it needs C2V_NUM_SAMPLED=<S>")
        if self._num_sampled and self.world > 1 and not self._sharded_sampled:
            raise ValueError("C2V_NUM_SAMPLED=%d: the sampled softmax trains on one GPU and this run has %d ranks; unset "
                             "C2V_NUM_SAMPLED to train on several GPUs, or train in a single process" % (
                                 self._num_sampled, self.world))
        if self._num_sampled and config.DL_FRAMEWORK == "b200-keras":
            raise ValueError("C2V_NUM_SAMPLED is not available with --framework b200-keras: its loss is the full-vocabulary "
                             "crossentropy; unset C2V_NUM_SAMPLED or train with --framework b200")
        # C2V_DEVICE_READER=1: train() reads its batches on the GPU (device_reader.py, DESIGN.md §6d)
        self._device_reader = device_reader_flag(os.environ)
        # C2V_SHARDED_READER=1: on several GPUs each rank reads and parses 1/W of every chunk (DESIGN.md §6d)
        self._sharded_reader = sharded_reader_flag(os.environ)
        self._reader_transport = None
        if self._sharded_reader and not self._device_reader:
            raise ValueError("C2V_SHARDED_READER=1 shards the device reader: it needs C2V_DEVICE_READER=1")
        if self._device_reader and config.DL_FRAMEWORK == "b200-keras":
            raise ValueError("C2V_DEVICE_READER=1 is not available with --framework b200-keras: its training loop reads "
                             "batches on the host; unset C2V_DEVICE_READER or train with --framework b200")
        # C2V_DEVICE_EVAL=1: evaluate() reads, predicts and scores on the GPU (device_reader.py, DESIGN.md §6e)
        self._device_eval = device_eval_flag(os.environ)
        if self._device_eval and config.DL_FRAMEWORK == "b200-keras":
            raise ValueError("C2V_DEVICE_EVAL=1 is not available with --framework b200-keras: its evaluation has its own "
                             "metrics and loss on the host; unset C2V_DEVICE_EVAL or evaluate with --framework b200")
        # C2V_DEVICE_TEXT=1: `.vectors` and word2vec files are formatted on the GPU (text_export.py, DESIGN.md §6f)
        self._device_text = device_text_flag(os.environ)
        # C2V_DEVICE_PREDICT=1: `--predict` reads, predicts and formats on the GPU (device_predict.py, DESIGN.md §6i)
        self._device_predict = device_predict_flag(os.environ)
        self._dev_predictor = None
        self._device_vocabs = None               # device_reader.DeviceVocabs, shared by the training and evaluation readers
        self._eval_tables = None                 # device_reader.eval_tables of the target vocabulary
        self._dev_eval_reader = None
        self._dev_corpus_reader = None           # C2V_DEVICE_EVAL=1: the reader of --score_names / --nearest's corpus
        self._dev_corpus_path = None
        if self.world > 1:
            self._join_group()
            if self.rank != 0:
                config.quiet()                       # rank 0 logs for every rank
        # C2V_EXTEND_VOCAB=1: --load with --data continues at the loaded vocabularies extended by the dataset's words
        self._extend_vocab = extend_vocab_run(config, extend_vocab_flag(os.environ), config.log)
        super().__init__(config)

    def _make_vocabs(self):
        from .vocabularies import Code2VecVocabs
        return Code2VecVocabs(self.config, extend=self._extend_vocab)

    def _join_group(self):
        import torch
        import torch.distributed as dist
        if not dist.is_initialized():
            torch.cuda.set_device(self.local_rank)
            dist.init_process_group("nccl", device_id=torch.device("cuda", self.local_rank))
            self._own_group = True
        if dist.get_world_size() != self.world:
            raise ValueError("WORLD_SIZE=%d but the process group has %d ranks" % (self.world, dist.get_world_size()))
        self.rank = dist.get_rank()

    def log(self, msg):
        if self.rank == 0:
            super().log(msg)

    def _all_ok(self, work, ranks=None):
        """work() on this rank if it is one of `ranks` (default: every rank), then every rank learns whether any rank
        failed, so all of them raise together instead of waiting in the next collective for a rank that has gone."""
        import torch.distributed as dist
        err = None
        if ranks is None or self.rank in ranks:
            try:
                work()
            except Exception as exc:
                err = exc
        status = [None] * self.world
        dist.all_gather_object(status, None if err is None else "%s: %s" % (type(err).__name__, err))
        if err is not None:
            raise err
        failed = [(r, s) for r, s in enumerate(status) if s]
        if failed:
            raise RuntimeError("rank %d failed: %s" % failed[0])

    def _init_num_of_examples(self):
        if self.world == 1:
            return super()._init_num_of_examples()
        # rank 0 counts the examples and writes the `.num_examples` side-cars; the other ranks then read them
        self._all_ok(super()._init_num_of_examples, ranks=(0,))
        if self.rank != 0:
            super()._init_num_of_examples()

    # ---- engine life cycle -------------------------------------------------------------------
    def _engine_dims(self) -> EngineDims:
        c = self.config
        if c.TOKEN_EMBEDDINGS_SIZE != c.PATH_EMBEDDINGS_SIZE:
            raise ValueError("the b200 backend needs TOKEN_EMBEDDINGS_SIZE == PATH_EMBEDDINGS_SIZE")
        if c.TARGET_EMBEDDINGS_SIZE != c.CODE_VECTOR_SIZE:
            raise ValueError("TARGET_EMBEDDINGS_SIZE must equal CODE_VECTOR_SIZE (logits = code_vectors . targets^T)")
        return EngineDims(token_vocab=self.vocabs.token_vocab.size, path_vocab=self.vocabs.path_vocab.size,
                          target_vocab=self.vocabs.target_vocab.size, embed_dim=c.TOKEN_EMBEDDINGS_SIZE,
                          code_dim=c.CODE_VECTOR_SIZE, max_contexts=c.MAX_CONTEXTS,
                          max_batch=max(c.TRAIN_BATCH_SIZE, c.TEST_BATCH_SIZE, 1),
                          top_k=c.TOP_K_WORDS_CONSIDERED_DURING_PREDICTION)

    def _checkpoint_dims(self, dims: dict) -> dict:
        """The model's dims `dims` (vars(EngineDims)) as a loaded checkpoint must have them: with C2V_EXTEND_VOCAB=1 the
        table sizes are the loaded vocabularies', whose rows are the leading rows of the grown tables."""
        if not self._extend_vocab:
            return dims
        sizes = self.vocabs.loaded_sizes
        return dict(dims, token_vocab=sizes[VocabType.Token], path_vocab=sizes[VocabType.Path],
                    target_vocab=sizes[VocabType.Target])

    def _make_engine(self, init: bool = False):
        """The engine and, for training or any multi-GPU run, its Trainer.  init: draw the initial parameters (on several
        GPUs before the Trainer moves the embedding tables into row shards)."""
        import torch
        Y = self.vocabs.target_vocab.size
        if self._num_sampled:
            check_num_sampled(self._num_sampled, Y)
        if self.config.is_training:
            self.log("b200 backend training loss: %s (C2V_NUM_SAMPLED=%d)" % (
                "sampled softmax, %d unique log-uniform negatives of the %d target words drawn on the GPU each step" % (
                    self._num_sampled, Y) if self._num_sampled else "full softmax over the %d target words" % Y,
                self._num_sampled))
        elif self._num_sampled:
            self.log("C2V_NUM_SAMPLED=%d has no effect: this run does not train (no --data)" % self._num_sampled)
        if self._sharded_sampled and self.world == 1:
            self.log("C2V_SHARDED_SAMPLED=1 has no effect on one GPU: the sampled softmax runs its one-GPU step")
        if self.world > 1:
            # this rank's engine: a block of target rows, sized for the global batch (trainer.make_fully_sharded_engine)
            self.engine = make_fully_sharded_engine(self._engine_dims(), self.config.TRAIN_BATCH_SIZE // self.world,
                                                    self.local_rank, training=self.config.is_training)
            if init:
                self.engine.init_params(scheme=self._INIT_SCHEME, whole_target_table=True)
        else:
            device = int(os.environ.get("LOCAL_RANK", "0")) if torch.cuda.device_count() > 1 else 0
            self.engine = PathAttentionEngine(self._engine_dims(), device=device, training=self.config.is_training)
        # arithmetic of the big matrix products: tensor cores (tf32 operands, fp32 accumulate) for training
        # steps, the reference's own fp32 FMA class for evaluate()/predict() so that top-k is decided on
        # fp32 logits.  C2V_MATH=fp32|tf32 forces one mode for both.
        forced = os.environ.get("C2V_MATH", "").lower()
        modes = {"fp32": 0, "tf32": 1, "3xtf32": 2}
        self._math_train = modes.get(forced, 1)
        # evaluate()/predict(): the tensor cores at fp32-equivalent accuracy (3xTF32), so top-k is decided on fp32-class
        # logits at tensor-core speed; both choices are logged, nothing switches silently
        self._math_eval = modes.get(forced, 2)
        self.log("b200 backend arithmetic: train = %s, evaluate/predict = %s (C2V_MATH=fp32|tf32|3xtf32 forces one for both)" % (
            {0: "fp32 FFMA", 1: "tf32 tensor cores", 2: "3xTF32 tensor cores (fp32-equivalent)"}[self._math_train],
            {0: "fp32 FFMA", 1: "tf32 tensor cores", 2: "3xTF32 tensor cores (fp32-equivalent)"}[self._math_eval]))
        # C2V_DETERMINISTIC / C2V_SEED: reproducible training runs (run_determinism)
        self._deterministic, self._seed = run_determinism(os.environ)
        if self.world > 1 and self._num_sampled:
            # every rank draws the sampled negatives from this seed, and a clock-derived one may differ between ranks
            import torch.distributed as dist
            seeds = [None] * self.world
            dist.all_gather_object(seeds, self._seed)
            self._seed = seeds[0]
        self.log("b200 backend run: deterministic = %d, seed = %d (C2V_DETERMINISTIC=%d C2V_SEED=%d replays it)" % (
            self._deterministic, self._seed, self._deterministic, self._seed))
        # C2V_HINT_NEXT=1: pass each next batch to the engine (c2v_hint_next_batch); off by default
        self._hint_next = os.environ.get("C2V_HINT_NEXT", "0") == "1"
        self.log("b200 backend training reader: %s (C2V_DEVICE_READER=%d)" % (
            "on the GPU" if self._device_reader else "on the host", self._device_reader))
        self.log(evaluation_route_line(self._device_eval))
        self.log("b200 backend text export: `.vectors` and word2vec files formatted %s (C2V_DEVICE_TEXT=%d)" % (
            "on the GPU" if self._device_text else "on the host", self._device_text))
        self.log("b200 backend predict: %s (C2V_DEVICE_PREDICT=%d)" % (
            "read, predicted in batches and formatted on the GPU" if self._device_predict else "one method at a time on the host",
            self._device_predict))
        if self.world > 1:
            # every multi-GPU run, evaluate-only ones too: the row shards and Trainer.predict live in the Trainer.
            # C2V_DETERMINISTIC=1 sends the embedding gradients through the ordered exchange (DESIGN.md §5.1)
            det = self._deterministic and self.config.is_training
            self.trainer = Trainer(self.engine, keep_prob=self.config.DROPOUT_KEEP_RATE, seed=self._seed, adam=self._ADAM,
                                   schedule="fully_sharded", deterministic=det, ordered_exchange=det)
            self.log("b200 backend: %d ranks, fully sharded schedule, %d of each global batch of %d rows per rank" % (
                self.world, self.engine.local_batch, self.config.TRAIN_BATCH_SIZE))
        elif self.config.is_training:
            self.trainer = Trainer(self.engine, keep_prob=self.config.DROPOUT_KEEP_RATE, seed=self._seed, adam=self._ADAM,
                                   deterministic=self._deterministic)
        if init and self.world == 1:
            self.engine.init_params(scheme=self._INIT_SCHEME)

    def _create_inner_model(self):
        self._make_engine(init=True)
        shapes = self._engine_dims().shapes()
        n_params = sum(int(np.prod(s)) for s in shapes.values())
        self.log("Number of trainable params: {}".format(n_params))
        for name, shape in shapes.items():
            self.log("variable name: {} -- shape: {} -- #params: {}".format(name, shape, int(np.prod(shape))))

    def _load_inner_model(self):
        """`X.c2v_b200` when it exists, else the TensorFlow checkpoint `X.index` + `X.data-*` when that exists, else the
        Keras backend's `X__only-weights` or `X__entire-model/` when one exists (_load_keras).  With C2V_EXTEND_VOCAB=1
        the engine is built at the merged vocabulary sizes and initialised as a model built from scratch at those sizes;
        the checkpoint, checked against the loaded sizes (_checkpoint_dims), then fills the leading rows."""
        if self._extend_vocab:
            self._make_engine(init=True)
        else:
            self._make_engine()
        load = self.config.MODEL_LOAD_PATH
        path = load + _CKPT_SUFFIX
        if not os.path.isfile(path) and os.path.isfile(load + INDEX_SUFFIX):
            self.log("Loading model weights from the TensorFlow checkpoint: " + load)
            (self._read_sharded_bundle if self.world > 1 else self._read_bundle)(load)
        elif not os.path.isfile(path) and (os.path.isfile(Config.get_model_weights_path(load) + INDEX_SUFFIX) or
                                           os.path.isdir(Config.get_entire_model_path(load))):
            self._load_keras(load)
        else:
            self.log("Loading model weights from: " + path)
            self._read_checkpoint(path)
        self.log("Done loading model weights")

    def close_session(self):
        if self._dev_predictor is not None:
            self._dev_predictor.close()
            self._dev_predictor = None
        if self._dev_eval_reader is not None:
            self._dev_eval_reader.close()
            self._dev_eval_reader = None
        if self._dev_corpus_reader is not None:
            self._dev_corpus_reader.close()
            self._dev_corpus_reader = None
        self._device_vocabs = None
        if getattr(self, "_knn_handle", None) is not None:
            self._knn_handle.close()
            self._knn_handle = None
        if self.engine is not None:
            if self.world > 1:
                import torch
                torch.cuda.synchronize(self.engine.dev)
                _barrier()                               # no peer reads this rank's shards any more
            self.engine.close()
            self.engine = None
        if self._reader_transport is not None:
            self._reader_transport.destroy()
            self._reader_transport = None
        if self._own_group:
            import torch.distributed as dist
            dist.destroy_process_group()
            self._own_group = False

    def save(self, model_save_path=None):
        if self.world == 1:
            return super().save(model_save_path)
        # rank 0 writes dictionaries.bin and makes the folder; every rank writes its rows of the checkpoint
        target = model_save_path if model_save_path is not None else self.config.MODEL_SAVE_PATH
        if self.rank == 0:
            folder = target.rpartition("/")[0]
            if folder:
                os.makedirs(folder, exist_ok=True)
            self.vocabs.save(self.config.get_vocabularies_path_from_model_path(target))
        self._save_inner_model(target)

    # ---- checkpoint: header (json) + raw little-endian float32 tensors -------------------------
    def _save_inner_model(self, path: str, release: bool = False):
        if self.world > 1:
            return self._save_sharded(path)
        if self._save_format == "tf":
            return self._save_bundle(path, release)
        if self._save_format == "keras":
            return self._save_keras(path, release or self.config.RELEASE)
        e = self.engine
        e.sync_tables()                                  # lazy Adam: replay deferred row updates before reading the tensors
        tensors = [e.params[k] for k in PARAM_NAMES]
        with_optimizer = (not release) and e.adam_m is not None
        if with_optimizer:
            tensors += [e.adam_m[k] for k in PARAM_NAMES] + [e.adam_v[k] for k in PARAM_NAMES]
        prefix, _, _ = checkpoint_header(vars(e.dims), e.adam_t, getattr(self, "nr_epochs_trained", 0), with_optimizer)
        tmp = path + _CKPT_SUFFIX + ".tmp"
        write_checkpoint(tmp, prefix, [t.detach().cpu().numpy() for t in tensors])
        os.replace(tmp, path + _CKPT_SUFFIX)

    def _sharded_tensors(self, with_optimizer: bool) -> dict:
        """{checkpoint tensor name: this rank's device tensor} (multi_rank's layout).  The replicated tok / path tensors
        are stale once the Trainer has moved them into row shards; only the shards are used."""
        e = self.engine
        out = {"theta/tok": e.shard_params["tok"], "theta/path": e.shard_params["path"]}
        out.update({"theta/" + k: e.params[k] for k in ("tgt", "W", "a")})
        if with_optimizer:
            for g, shard, rest in (("adam_m", e.shard_m, e.adam_m), ("adam_v", e.shard_v, e.adam_v)):
                out.update({g + "/tok": shard["tok"], g + "/path": shard["path"]})
                out.update({g + "/" + k: rest[k] for k in ("tgt", "W", "a")})
        return out

    def _save_sharded(self, path: str):
        """All ranks write one file: rank 0 writes the header and sizes the file, every rank writes its own rows
        (embedding-shard rows, its target block; W and a from rank 0), rank 0 renames the file once all are done."""
        e = self.engine
        with_optimizer = e.adam_m is not None
        prefix, entries, total = checkpoint_header(vars(self._engine_dims()), e.adam_t,
                                                   getattr(self, "nr_epochs_trained", 0), with_optimizer)
        tmp = path + _CKPT_SUFFIX + ".tmp"
        rows = (e.target_row0, e.target_row0 + e.dims.target_vocab)

        def write_rows():
            local = {name: t.detach().cpu().numpy() for name, t in self._sharded_tensors(with_optimizer).items()
                     if self.rank == 0 or name.split("/")[1] not in ("W", "a")}
            write_checkpoint_part(tmp, len(prefix), entries, self.rank, self.world, rows, local)
        # each step ends in a collective that also reports a failure on any rank, so no rank waits for one that has gone
        self._all_ok(lambda: create_checkpoint_file(tmp, prefix, total), ranks=(0,))
        self._all_ok(write_rows)
        self._all_ok(lambda: os.replace(tmp, path + _CKPT_SUFFIX), ranks=(0,))     # the file exists on return, on any rank

    def _read_sharded(self, file_path: str):
        """This rank's rows of a checkpoint saved on any number of GPUs, into the shards, the target block and W / a
        (with the Adam slots when training, so a resumed run continues exactly).  Runs after the Trainer is built:
        enable_table_sharding would overwrite the shards and zero their Adam slots."""
        import torch
        e = self.engine

        def read_rows():
            out = self._sharded_tensors(with_optimizer=e.training)
            check_checkpoint_dims(read_checkpoint_header(file_path)[0], self._checkpoint_dims(vars(self._engine_dims())))
            meta = read_checkpoint_part(file_path, self.rank, self.world,
                                        (e.target_row0, e.target_row0 + e.dims.target_vocab), out)
            e.adam_t = int(meta.get("adam_t", 0))
            if e.training:
                e.set_option("adam_step_count", e.adam_t)
            torch.cuda.synchronize(e.dev)
        self._all_ok(read_rows)                          # every shard is loaded before any peer reads it

    # ---- TensorFlow V2 checkpoints (tf_bundle.py, DESIGN.md §6k) -------------------------------------------------
    def _adam_betas(self):
        adam = self._ADAM or ADAM_DEFAULTS
        return adam["beta1"], adam["beta2"]

    def _set_adam_t(self, adam_t: int):
        e = self.engine
        e.adam_t = int(adam_t)
        if e.training:
            e.set_option("adam_step_count", e.adam_t)

    @staticmethod
    def _check_crcs(entries, computed) -> None:
        """ValueError naming the first tensor whose device CRC-32C (computed, device int32 [n]) is not the stored one."""
        got = computed.cpu().numpy().view(np.uint32)
        for ent, c in zip(entries, got):
            if int(c) != ent["crc"]:
                raise ValueError("checkpoint tensor %s fails its CRC-32C: stored 0x%08x, computed 0x%08x" % (
                    ent["key"], ent["crc"], int(c)))

    def _read_bundle(self, prefix: str):
        """The bundle's tensors streamed through page-locked staging into the engine's tensors, each tensor's CRC-32C
        computed on the device as its rows arrive, then all compared with the stored ones."""
        import torch
        e = self.engine
        entries, adam_t = bundle_entries(prefix, self._checkpoint_dims(vars(e.dims)), e.adam_m is not None, *self._adam_betas())
        dest = {"theta": e.params, "adam_m": e.adam_m, "adam_v": e.adam_v}
        computed = torch.empty(len(entries), dtype=torch.int32, device=e.dev)
        with torch.cuda.device(e.dev), _PinnedStaging(e.dev) as stage:
            for i, ent in enumerate(entries):
                group, name = ent["name"].split("/")
                t = _lead(dest[group][name], ent["shape"])
                stage.upload(ent["file"], ent["offset"], ent["nbytes"], t)
                tensor_crc32c(t, *crc_view(name, ent["shape"]), computed[i:i + 1])
        self._check_crcs(entries, computed)
        self._set_adam_t(adam_t)

    def _read_sharded_bundle(self, prefix: str):
        """_read_sharded for a bundle: every rank reads its own rows, computes their CRC-32Cs on its device, gathers the
        row CRCs of the sharded tables into global row order and combines them; a failure on any rank (a tensor missing,
        a wrong shape, a CRC mismatch) raises on every rank."""
        import torch
        import torch.distributed as dist
        e = self.engine
        W, r = self.world, self.rank
        state = {}

        def read_rows():
            entries, adam_t = bundle_entries(prefix, self._checkpoint_dims(vars(self._engine_dims())), e.training, *self._adam_betas())
            out = self._sharded_tensors(with_optimizer=e.training)
            read_entries_part(prefix, 0, entries, r, W, (e.target_row0, e.target_row0 + e.dims.target_vocab), out)
            torch.cuda.synchronize(e.dev)
            state.update(entries=entries, out=out, adam_t=adam_t)
        self._all_ok(read_rows)                          # every shard is loaded before any peer reads it
        entries, out = state["entries"], state["out"]
        computed = torch.empty(len(entries), dtype=torch.int32, device=e.dev)
        with torch.cuda.device(e.dev):
            for i, ent in enumerate(entries):
                name = ent["name"].split("/")[1]
                rows, row_bytes = crc_view(name, ent["shape"])
                t = out[ent["name"]]
                if name in ("W", "a"):                   # replicated: every rank checks its own copy
                    tensor_crc32c(t, rows, row_bytes, computed[i:i + 1])
                    continue
                # tok / path: local row i is global row i * W + r (ceil(T / W) rows per rank, padding past the end);
                # tgt: rank r's block of ceil(Y / W) rows (the last one shorter), padded to that length.  Y is the engine's:
                # with C2V_EXTEND_VOCAB=1 the stored rows are the first `rows` of the grown table
                per = int(t.shape[0]) if name != "tgt" else -(-e.global_target_vocab // W)
                local = torch.zeros(per, dtype=torch.int32, device=e.dev)
                n_own = min(per, int(t.shape[0]))
                crc32c_rows(t, n_own, row_bytes, row_bytes, local)
                gathered = torch.empty(W * per, dtype=torch.int32, device=e.dev)
                dist.all_gather_into_tensor(gathered, local)
                order = gathered.view(W, per).t() if name != "tgt" else gathered.view(W, per)
                crc32c_combine(order.reshape(-1)[:rows].contiguous(), rows, row_bytes, computed[i:i + 1])
        self._all_ok(lambda: self._check_crcs(entries, computed))
        self._set_adam_t(state["adam_t"])

    def _save_bundle(self, path: str, release: bool):
        """<path>.index + <path>.data-00000-of-00001: every tensor's CRC-32C computed on the device, then its bytes
        downloaded through page-locked staging into the data file, in key order; the Adam beta powers for e.adam_t."""
        import torch
        e = self.engine
        e.sync_tables()                                  # lazy Adam: replay deferred row updates before reading the tensors
        with_optimizer = (not release) and e.adam_m is not None
        tensors, scalars = bundle_layout(vars(e.dims), with_optimizer, e.adam_t, *self._adam_betas())
        src = {"theta": e.params, "adam_m": e.adam_m, "adam_v": e.adam_v}
        dev = [src[n.split("/")[0]][n.split("/")[1]] for _, n, _, _, _ in tensors]
        computed = torch.empty(max(len(tensors), 1), dtype=torch.int32, device=e.dev)
        tmp = data_file(path) + ".tmp"
        with torch.cuda.device(e.dev):
            for i, ((_, name, shape, _, _), t) in enumerate(zip(tensors, dev)):
                tensor_crc32c(t, *crc_view(name.split("/")[1], t.shape), computed[i:i + 1])
            crcs = computed.cpu().numpy().view(np.uint32)
            pieces = [(off, t) for (_, _, _, off, _), t in zip(tensors, dev)]
            pieces += [(off, np.asarray(v, dtype="<f4")) for _, v, off in scalars]
            with open(tmp, "wb") as f, _PinnedStaging(e.dev) as stage:
                for off, t in sorted(pieces, key=lambda p: p[0]):
                    if isinstance(t, np.ndarray):
                        f.write(t.tobytes())
                    else:
                        stage.download(t, f)
        index = [(key, shape, off, n, int(c)) for (key, _, shape, off, n), c in zip(tensors, crcs)]
        index += [(key, (), off, 4, host_crc32c(np.asarray(v, dtype="<f4").tobytes())) for key, v, off in scalars]
        os.replace(tmp, data_file(path))
        write_index(path, index)

    # ---- the reference Keras backend's checkpoints (keras_ckpt.py, DESIGN.md §6l) --------------------------------
    def _load_keras(self, load: str):
        """The rule of the reference's Keras backend (keras_model.py:241-280): training needs the entire model; otherwise
        the weights file when it exists, else the latest checkpoint of the entire model, whose `ckpt-N` gives the epochs
        trained."""
        entire, weights = Config.get_entire_model_path(load), Config.get_model_weights_path(load)
        must_use_entire_model = self.config.is_training
        entire_model_exists = os.path.exists(entire)
        model_weights_exist = os.path.isfile(weights + INDEX_SUFFIX)
        if must_use_entire_model and not entire_model_exists:
            raise ValueError(
                "There is no model at path `{model_file_path}`. When loading the model for further training, "
                "we must use an entire saved model file (not just weights).".format(model_file_path=entire))
        if not entire_model_exists and not model_weights_exist:
            raise ValueError(
                "There is no entire model to load at path `{entire_model_path}`, "
                "and there is no model weights file to load at path `{model_weights_path}`.".format(
                    entire_model_path=entire, model_weights_path=weights))
        if self.world > 1:
            raise ValueError("`%s`: Keras checkpoints are read by one GPU; convert it once in a single process (without "
                             "torch.distributed.run), e.g. `--load %s --save <X>` saves a .c2v_b200 checkpoint that loads on "
                             "any number of GPUs" % (load, load))
        if must_use_entire_model or not model_weights_exist:
            self.log("Loading entire model from path `{}`.".format(entire))
            latest = latest_checkpoint(entire)
            if latest is None:
                raise ValueError("Failed to load model: Model latest checkpoint is not found.")
            self.log("Loading latest checkpoint `{}`.".format(latest))
            self._read_keras(latest)
            if hasattr(self, "nr_epochs_trained"):           # the Keras-schedule backend resumes at this epoch
                self.nr_epochs_trained = int(latest.split("-")[-1])
        else:
            self.log("Loading model weights from path `{}`.".format(weights))
            self._read_keras(weights)

    def _chunk_rows(self, Y: int) -> int:
        """File rows of a [D, Y] kernel per device chunk: whole rows, at most _PinnedStaging.CHUNK_BYTES unless one row
        is larger."""
        return max(1, _PinnedStaging.CHUNK_BYTES // (4 * Y))

    def _read_keras(self, prefix: str):
        """As _read_bundle; the [D, Y] output kernel (and its slots) goes through one device chunk of whole file rows:
        each chunk's row CRCs in file order, then c2v_rows_to_cols into the engine's [Y, D] tensor."""
        import torch
        e = self.engine
        entries, adam_t, self._keras_save_counter = keras_entries(prefix, self._checkpoint_dims(vars(e.dims)), e.adam_m is not None,
                                                                  self._ADAM or ADAM_DEFAULTS)
        dest = {"theta": e.params, "adam_m": e.adam_m, "adam_v": e.adam_v}
        computed = torch.empty(len(entries), dtype=torch.int32, device=e.dev)
        with torch.cuda.device(e.dev), _PinnedStaging(e.dev) as stage:
            chunk = row_crc = None
            for i, ent in enumerate(entries):
                group, name = ent["name"].split("/")
                t = _lead(dest[group][name], ent["shape"])
                if not ent["transposed"]:
                    stage.upload(ent["file"], ent["offset"], ent["nbytes"], t)
                    tensor_crc32c(t, *crc_view(name, ent["shape"]), computed[i:i + 1])
                    continue
                Y, D = t.shape
                rows = min(self._chunk_rows(Y), D)
                if chunk is None:
                    chunk = torch.empty(rows * Y, dtype=torch.float32, device=e.dev)
                    row_crc = torch.empty(D, dtype=torch.int32, device=e.dev)
                for i0 in range(0, D, rows):
                    k = min(rows, D - i0)
                    stage.upload(ent["file"], ent["offset"] + i0 * 4 * Y, k * 4 * Y, chunk[:k * Y])
                    crc32c_rows(chunk, k, 4 * Y, 4 * Y, row_crc[i0:i0 + k])
                    rows_to_cols(chunk, k, Y, t, i0)
                crc32c_combine(row_crc, D, 4 * Y, computed[i:i + 1])
        self._check_crcs(entries, computed)
        self._set_adam_t(adam_t)

    def _save_keras(self, path: str, release: bool):
        """`path__only-weights` (release: the weights alone) or `path__entire-model/ckpt-<epochs trained>` with the
        optimizer, then the manager's state file and MAX_TO_KEEP rotation.  Each tensor's CRC-32C is computed on the
        device; the [D, Y] output kernel is gathered into one device chunk of whole file rows at a time
        (c2v_cols_to_rows), checked and downloaded."""
        import torch
        e = self.engine
        e.sync_tables()                                  # lazy Adam: replay deferred row updates before reading the tensors
        with_optimizer = (not release) and e.adam_m is not None
        self._keras_save_counter = getattr(self, "_keras_save_counter", 0) + (0 if release else 1)
        if release:
            prefix = Config.get_model_weights_path(path)
        else:
            directory = Config.get_entire_model_path(path)
            os.makedirs(directory, exist_ok=True)
            prefix = os.path.join(directory, "ckpt-%d" % getattr(self, "nr_epochs_trained", 0))
        tensors, scalars = keras_layout(vars(e.dims), not release, with_optimizer, e.adam_t, self._keras_save_counter,
                                        self._ADAM or ADAM_DEFAULTS)
        src = {"theta": e.params, "adam_m": e.adam_m, "adam_v": e.adam_v}
        pieces = [(off, src[n.split("/")[0]][n.split("/")[1]], i) for i, (_, n, _, off, _) in enumerate(tensors)]
        pieces += [(off, raw, None) for _, _, _, raw, off, _ in scalars]
        computed = torch.empty(max(len(tensors), 1), dtype=torch.int32, device=e.dev)
        tmp = data_file(prefix) + ".tmp"
        with torch.cuda.device(e.dev), open(tmp, "wb") as f, _PinnedStaging(e.dev) as stage:
            chunk = row_crc = None
            for _, t, i in sorted(pieces, key=lambda p: p[0]):
                if i is None:
                    f.write(t)
                elif tensors[i][1].split("/")[1] != "tgt":
                    tensor_crc32c(t, *crc_view(tensors[i][1].split("/")[1], t.shape), computed[i:i + 1])
                    stage.download(t, f)
                else:
                    Y, D = t.shape
                    rows = min(self._chunk_rows(Y), D)
                    if chunk is None:
                        chunk = torch.empty(rows * Y, dtype=torch.float32, device=e.dev)
                        row_crc = torch.empty(D, dtype=torch.int32, device=e.dev)
                    for i0 in range(0, D, rows):
                        k = min(rows, D - i0)
                        cols_to_rows(t, i0, k, Y, chunk)
                        crc32c_rows(chunk, k, 4 * Y, 4 * Y, row_crc[i0:i0 + k])
                        stage.download(chunk[:k * Y], f)
                    crc32c_combine(row_crc, D, 4 * Y, computed[i:i + 1])
            crcs = computed.cpu().numpy().view(np.uint32)
        os.replace(tmp, data_file(prefix))
        write_keras_index(prefix, tensors, scalars, crcs)
        if not release:
            record_checkpoint(directory, prefix, self.config.MAX_TO_KEEP, time.time())

    def _read_checkpoint(self, file_path: str):
        import torch
        if self.world > 1:
            return self._read_sharded(file_path)
        if not os.path.isfile(file_path):
            raise ValueError("There is no model at path `{}`.".format(file_path))
        e = self.engine
        with open(file_path, "rb") as f:
            if f.read(8) != _CKPT_MAGIC:
                raise ValueError("`{}` is not a c2v_b200 checkpoint".format(file_path))
            (hlen,) = struct.unpack("<Q", f.read(8))
            meta = json.loads(f.read(hlen).decode())
            base = f.tell()
            want = self._checkpoint_dims(vars(e.dims))
            for key in ("token_vocab", "path_vocab", "target_vocab", "embed_dim", "code_dim"):
                if meta["dims"][key] != want[key]:
                    raise ValueError("checkpoint %s=%s does not match the model (%s)" % (key, meta["dims"][key], want[key]))
            dest = {"theta": e.params, "adam_m": e.adam_m, "adam_v": e.adam_v}
            for ent in meta["tensors"]:
                group, name = ent["name"].split("/")
                if dest.get(group) is None:
                    continue
                f.seek(base + ent["offset"])
                arr = np.frombuffer(f.read(ent["nbytes"]), dtype="<f4").reshape(ent["shape"])
                _lead(dest[group][name], ent["shape"]).copy_(torch.from_numpy(arr.copy()))
            e.adam_t = int(meta.get("adam_t", 0))
            if e.training:
                # resuming: the engine's own step counter (lazy Adam needs consecutive steps and marks every row
                # as current as of this step) has to agree with the restored optimizer state
                e.set_option("adam_step_count", e.adam_t)
            if hasattr(self, "nr_epochs_trained"):           # the Keras-schedule backend resumes at this epoch
                self.nr_epochs_trained = int(meta.get("epochs_trained", 0))

    # ---- train (tensorflow_model.py:40-112) ------------------------------------------------------
    def train(self):
        self.log("Starting training")
        start_time = time.time()
        cfg = self.config
        batch_num, sum_loss = 0, 0.0
        multi_batch_start_time = time.time()
        num_batches_to_save_and_eval = max(int(cfg.train_steps_per_epoch * cfg.SAVE_EVERY_EPOCHS), 1)
        train_reader = PathContextReader(vocabs=self.vocabs, model_input_tensors_former=_TrainInputFormer(),
                                         config=cfg, estimator_action=EstimatorAction.Train, shuffle_seed=self._seed)
        self.log("Started reader...")
        former = _TrainInputFormer()
        # pinned-host batch ring + copy stream (batch_ring.py): the reader thread draws every batch straight into a
        # page-locked slot, its upload overlaps the previous step, and the loop never waits for the GPU except to read
        # the losses at each progress line.  C2V_BATCH_RING=0 (or a reader without the native tensoriser) keeps the
        # synchronous c2v_train_batch_host path.
        # several GPUs: every rank reads the same global batches (same file, same shuffle seed) and steps on its slice
        multi = self.world > 1
        num_sampled = self._num_sampled        # > 0: every step is Trainer.step_sampled (several ranks: C2V_SHARDED_SAMPLED=1)
        dropped_rows = 0
        ring = dev_reader = None
        if self._device_reader:
            # C2V_DEVICE_READER=1: batches are parsed and drawn on the GPU into device slots (device_reader.py); the steps
            # read them there (step_device) and the losses collect in the pinned history, as on the ring path
            from .device_reader import DeviceBatchReader
            if self._sharded_reader and multi:
                # C2V_SHARDED_READER=1: each rank reads 1/W of every chunk; the ranks meet once per chunk on a gloo group
                # of the reader's own (device_reader.make_share_transport), closed in close_session()
                if self._reader_transport is None:
                    self._reader_transport = _device_reader_mod.make_share_transport(self.engine.dev.index or 0)
                self.log("Training reader sharded across %d ranks: each reads and parses 1/%d of every chunk" % (
                    self.world, self.world))
            elif self._sharded_reader:
                self.log("C2V_SHARDED_READER=1 has no effect on one GPU: the device reader reads the whole file")
            dev_reader = DeviceBatchReader(train_reader, self.engine.dev, world=self.world, rank=self.rank,
                                           transport=self._reader_transport if multi else None,
                                           vocabs=self._shared_device_vocabs(train_reader))
        elif not multi and os.environ.get("C2V_BATCH_RING", "1") != "0" and not self._hint_next and train_reader._native_ready():
            import torch
            from .batch_ring import PinnedBatchRing
            ring = PinnedBatchRing(torch, self.engine.dev, cfg.TRAIN_BATCH_SIZE, cfg.MAX_CONTEXTS)
            train_reader.batch_ring = ring
        if ring is not None or dev_reader is not None:
            import torch
            loss_hist = torch.zeros(max(int(cfg.NUM_BATCHES_TO_LOG_PROGRESS), 1), dtype=torch.float32).pin_memory()
            n_hist = 0
        # the losses of a device-reader run are summed as the host path it replaces sums them: the ring path adds a float32
        # sum of the history, the synchronous path (C2V_HINT_NEXT=1, several GPUs) adds each step's loss in turn
        ring_sum = dev_reader is not None and not multi and not self._hint_next
        self.h2d_bytes = 0
        batches = dev_reader if dev_reader is not None else _prefetch(train_reader.get_dataset(), depth=4 if ring else 8)
        for batch, following in _with_next(batches):
            if dev_reader is not None:
                batch.wait()                       # the current stream waits for the draw into this slot
                if multi:
                    dropped_rows += batch.dropped
                    if batch.hi == batch.lo:       # fewer rows than ranks: the batch is skipped
                        batch.release()
                        continue
                nxt = None
                if self._hint_next and not multi and following is not None and not num_sampled:
                    following.wait()
                    nxt = following.tensors[:3]
                batch_num += 1
                self.engine.set_option("math_mode", self._math_train)
                if num_sampled:
                    loss = self.trainer.step_sampled(*batch.tensors, num_sampled)
                else:
                    loss = self.trainer.step_device(*batch.tensors, next_batch=nxt)
                batch.release()                    # the slot is reused once this step has run
                loss_hist[n_hist:n_hist + 1].copy_(loss, non_blocking=True)
                n_hist += 1
                flush = (batch_num % cfg.NUM_BATCHES_TO_LOG_PROGRESS == 0) or (batch_num % num_batches_to_save_and_eval == 0) \
                    or n_hist == loss_hist.numel()
                batch_loss = 0.0
                if flush:
                    torch.cuda.current_stream(self.engine.dev).synchronize()
                    if ring_sum:
                        batch_loss = float(loss_hist[:n_hist].sum())
                    else:
                        for v in loss_hist[:n_hist].tolist():
                            sum_loss += v
                    n_hist = 0
            else:
                t = former.from_model_input_form(batch)
                if multi:
                    # a short last batch runs as a step of world * floor(rows / world) rows (the loss is their mean)
                    lo, hi, dropped = batch_split(int(t.target_index.shape[0]), self.world, self.rank)
                    dropped_rows += dropped
                    if hi == lo:                       # fewer rows than ranks: the batch is skipped
                        continue
                nxt = None
                if self._hint_next and not multi and following is not None and not num_sampled:
                    n = former.from_model_input_form(following)
                    nxt = (n.path_source_token_indices, n.path_indices, n.path_target_token_indices)
                batch_num += 1
                self.engine.set_option("math_mode", self._math_train)
                if ring is not None:
                    rows = int(t.target_index.shape[0])
                    if num_sampled:                    # upload, draw and step queued; nothing waited for
                        dev, slot = ring.upload_next(rows)
                        loss = self.trainer.step_sampled(dev["src"], dev["path"], dev["tgt"], dev["mask"], dev["target"],
                                                         num_sampled)
                        ring.mark_compute_done(slot)
                        loss_hist[n_hist:n_hist + 1].copy_(loss, non_blocking=True)
                    else:
                        self.trainer.step_ring(ring, rows, loss_hist[n_hist:n_hist + 1])      # upload + step queued; nothing waited for
                    n_hist += 1
                    self.h2d_bytes += rows * (4 * cfg.MAX_CONTEXTS + 1) * 4
                    flush = (batch_num % cfg.NUM_BATCHES_TO_LOG_PROGRESS == 0) or (batch_num % num_batches_to_save_and_eval == 0) \
                        or n_hist == loss_hist.numel()
                    batch_loss = 0.0
                    if flush:                          # the losses of the steps since the last progress line reach the host here
                        torch.cuda.current_stream(self.engine.dev).synchronize()
                        batch_loss = float(loss_hist[:n_hist].sum())
                        n_hist = 0
                elif multi:                            # the fully sharded loss is already the mean over the global batch
                    rows = tuple(a[lo:hi] for a in (t.path_source_token_indices, t.path_indices, t.path_target_token_indices,
                                                    t.context_valid_mask, t.target_index))
                    if num_sampled:
                        batch_loss = self.trainer.step_host_sampled(*rows, num_sampled)
                    else:
                        batch_loss = self.trainer.step_host(*rows)
                elif num_sampled:
                    batch_loss = self.trainer.step_host_sampled(t.path_source_token_indices, t.path_indices,
                                                                t.path_target_token_indices, t.context_valid_mask,
                                                                t.target_index, num_sampled)
                else:
                    batch_loss = self.trainer.step_host(t.path_source_token_indices, t.path_indices, t.path_target_token_indices,
                                                        t.context_valid_mask, t.target_index, next_batch=nxt)
            sum_loss += batch_loss
            if batch_num % cfg.NUM_BATCHES_TO_LOG_PROGRESS == 0:
                if num_sampled:
                    self._check_sampler()
                self._trace_training(sum_loss, batch_num, multi_batch_start_time)
                sum_loss = 0.0
                multi_batch_start_time = time.time()
            if batch_num % num_batches_to_save_and_eval == 0:
                epoch_num = int((batch_num / num_batches_to_save_and_eval) * cfg.SAVE_EVERY_EPOCHS)
                if cfg.MODEL_SAVE_PATH:
                    model_save_path = cfg.MODEL_SAVE_PATH + "_iter" + str(epoch_num)
                    self.save(model_save_path)
                    self.log("Saved after %d epochs in: %s" % (epoch_num, model_save_path))
                if cfg.is_testing:
                    results = self.evaluate()
                    text = str(results).replace("topk", "top{}".format(cfg.TOP_K_WORDS_CONSIDERED_DURING_PREDICTION))
                    self.log("After {nr_epochs} epochs -- {evaluation_results}".format(nr_epochs=epoch_num, evaluation_results=text))
        if ring is not None:
            import torch
            torch.cuda.current_stream(self.engine.dev).synchronize()
            if n_hist:
                sum_loss += float(loss_hist[:n_hist].sum())
            ring.close()
            train_reader.batch_ring = None
        if dev_reader is not None:
            torch.cuda.current_stream(self.engine.dev).synchronize()
            if ring_sum:
                sum_loss += float(loss_hist[:n_hist].sum()) if n_hist else 0.0
            else:
                for v in loss_hist[:n_hist].tolist():
                    sum_loss += v
            self.h2d_bytes = dev_reader.h2d_bytes
            peers = "" if dev_reader.transport is None else ", %.1f MB of rows read from peers" % (dev_reader.peer_bytes / 1e6)
            self.log("Device reader: %.1f MB of text and draw indices uploaded, %.1f MB of device memory held%s" % (
                dev_reader.h2d_bytes / 1e6, dev_reader.device_bytes() / 1e6, peers))
            dev_reader.close()
        if num_sampled:
            self._check_sampler()
        if multi:
            self.log("%d training rows left out: a short batch trains on a multiple of the %d ranks" % (
                dropped_rows, self.world))
        self.log("Done training")
        if cfg.MODEL_SAVE_PATH:
            self.save(cfg.MODEL_SAVE_PATH)
            self.log("Model saved in file: %s" % cfg.MODEL_SAVE_PATH)
        elapsed = int(time.time() - start_time)
        self.log("Training time: %sH:%sM:%sS\n" % ((elapsed // 60 // 60), (elapsed // 60) % 60, elapsed % 60))

    def _check_sampler(self):
        """RuntimeError if a sampled step's draw reached the sampler's cap of 2^31 draws without num_sampled distinct
        classes (engine option "sampler_cap_hits"; the read synchronises, so it is made where train() waits anyway)."""
        hits = self.engine.get_option("sampler_cap_hits")
        if hits:
            raise RuntimeError("the log-uniform sampler reached its cap of 2^31 draws without %d distinct classes in %d "
                               "step(s)" % (self._num_sampled, hits))

    # ---- evaluate (tensorflow_model.py:114-195) ------------------------------------------------------
    def evaluate(self) -> Optional[ModelEvaluationResults]:
        eval_start_time = time.time()
        cfg = self.config
        if self.eval_reader is None:
            self.eval_reader = PathContextReader(vocabs=self.vocabs, model_input_tensors_former=_EvaluateInputFormer(),
                                                 config=cfg, estimator_action=EstimatorAction.Evaluate)
        if cfg.MODEL_LOAD_PATH and not cfg.TRAIN_DATA_PATH_PREFIX and cfg.RELEASE:
            release_name = cfg.MODEL_LOAD_PATH + ".release"
            self.log("Releasing model, output model: %s" % release_name)
            self._save_inner_model(release_name, release=True)
            return None                            # as the reference does after --release (:132-136)
        self.engine.set_option("math_mode", self._math_eval)
        special = self.vocabs.target_vocab.special_words
        subtokens_metric = SubtokensEvaluationMetric(partial(common.filter_impossible_names, special))
        topk_metric = TopKAccuracyEvaluationMetric(cfg.TOP_K_WORDS_CONSIDERED_DURING_PREDICTION,
                                                   partial(common.get_first_match_word_from_top_predictions, special))
        if self._device_eval:
            return self._evaluate_device(eval_start_time, subtokens_metric, topk_metric)
        total_predictions, total_batches = 0, 0
        # several GPUs: every rank predicts its slice of each batch, rank 0 gathers the rows and writes every file
        writer = self.rank == 0
        code_vectors_file, text = self._open_code_vectors(writer)
        with (open("log.txt", "w") if writer else contextlib.nullcontext()) as log_output_file:
            start_time = time.time()
            self.log("Starting evaluation")
            for batch in _prefetch(self.eval_reader.get_dataset()):
                t = _EvaluateInputFormer().from_model_input_form(batch)
                if self.world > 1:
                    idx, code_vectors = self._predict_sharded(t, cfg.EXPORT_CODE_VECTORS)
                    if not writer:
                        continue
                else:
                    idx, _vals, code_vectors, _attn = self.engine.predict_batch_host(
                        t.path_source_token_indices, t.path_indices, t.path_target_token_indices, t.context_valid_mask,
                        normalize=False, want_code=cfg.EXPORT_CODE_VECTORS, want_attention=False)
                top_words = self.vocabs.target_vocab.lookup_word(idx)          # (batch, top_k) strings   (:302)
                original_names = list(t.target_string)
                self._log_predictions_during_evaluation(zip(original_names, top_words), log_output_file)
                topk_metric.update_batch(zip(original_names, top_words))
                subtokens_metric.update_batch(zip(original_names, top_words))
                total_predictions += len(original_names)
                total_batches += 1
                if code_vectors_file is not None:
                    self._export_code_vectors(code_vectors_file, text, code_vectors)
                if total_batches % cfg.NUM_BATCHES_TO_LOG_PROGRESS == 0:
                    self._trace_evaluation(total_predictions, time.time() - start_time)
            self.log("Done evaluating, epoch reached")
            if writer:
                log_output_file.write(str(topk_metric.topk_correct_predictions) + "\n")
        if code_vectors_file is not None:
            self._close_code_vectors(code_vectors_file, text)
        elapsed = int(time.time() - eval_start_time)
        self.log("Evaluation time: %sH:%sM:%sS" % ((elapsed // 60 // 60), (elapsed // 60) % 60, elapsed % 60))
        results = None
        if writer:
            results = ModelEvaluationResults(topk_acc=topk_metric.topk_correct_predictions,
                                             subtoken_precision=subtokens_metric.precision,
                                             subtoken_recall=subtokens_metric.recall, subtoken_f1=subtokens_metric.f1)
        if self.world > 1:                         # every rank returns rank 0's results
            import torch.distributed as dist
            gathered = [None] * self.world
            dist.all_gather_object(gathered, results)
            results = gathered[0]
        return results

    # ---- evaluate on the GPU (C2V_DEVICE_EVAL=1, DESIGN.md §6e) -------------------------------------------------------
    def _shared_device_vocabs(self, reader: PathContextReader):
        """The model's vocabularies on its device, uploaded once and shared by its training and evaluation readers."""
        if self._device_vocabs is None:
            from .device_reader import DeviceVocabs
            reader.use_native = True
            reader._native_ready()                 # RuntimeError when libc2v_batcher.so cannot be built
            self._device_vocabs = DeviceVocabs(reader, self.engine.dev)
        return self._device_vocabs

    def _device_eval_reader(self):
        """The evaluation reader on the GPU, made once per model (and again after a pass that failed)."""
        if self._dev_eval_reader is None:
            from .device_reader import DeviceBatchReader, eval_tables
            reader = PathContextReader(vocabs=self.vocabs, model_input_tensors_former=_EvaluateInputFormer(),
                                       config=self.config, estimator_action=EstimatorAction.Evaluate)
            if self._eval_tables is None:
                self._eval_tables = eval_tables(self.vocabs.target_vocab)
            self._dev_eval_reader = DeviceBatchReader(reader, self.engine.dev, vocabs=self._shared_device_vocabs(reader),
                                                      tables=self._eval_tables)
        return self._dev_eval_reader

    def _evaluate_device(self, eval_start_time, subtokens_metric, topk_metric) -> Optional[ModelEvaluationResults]:
        """evaluate() with the test file read, predicted and scored on the GPU: the same results, log.txt and .vectors
        as the host route.  Rows the metric kernel flags (a name with a byte >= 0x80, or a top-k without a legal word)
        are scored by the host metrics themselves; the device's integer sums of the other rows are added to the same
        metric objects, whose properties then compute every float."""
        cfg = self.config
        top_k = cfg.TOP_K_WORDS_CONSIDERED_DURING_PREDICTION
        index_to_word = self.vocabs.target_vocab.index_to_word
        hist = np.zeros(top_k, dtype=np.int64)
        counts = np.zeros(4, dtype=np.int64)          # rows, tp, fp, fn of the rows scored on the device
        total_predictions, total_batches = 0, 0
        writer = self.rank == 0
        reader = self._device_eval_reader()
        code_vectors_file, text = self._open_code_vectors(writer)
        try:
            with (open("log.txt", "w") if writer else contextlib.nullcontext()) as log_output_file:
                start_time = time.time()
                self.log("Starting evaluation")
                for batch in reader:
                    batch.wait()                   # the current stream waits for the take into this slot
                    n = batch.hi - batch.lo
                    if self.world > 1:
                        ids, code = self._predict_sharded_device(batch.tensors[:4], n, cfg.EXPORT_CODE_VECTORS)
                    else:
                        code, _ = self.engine.forward(*batch.tensors[:4], want_attention=False)
                        ids, _ = self.engine.topk(code, normalize=False)
                    if writer:
                        sc = reader.score(batch, ids)              # synchronises the current stream
                        if code_vectors_file is not None:
                            code_vectors = code if text is not None else code.cpu().numpy()
                    batch.release()
                    total_predictions += n
                    total_batches += 1
                    if writer:
                        k = sc.acc.size - 4
                        hist[:k] += sc.acc[:k]
                        counts += sc.acc[k:]
                        self._log_and_score_host_rows(sc, n, index_to_word, log_output_file, subtokens_metric,
                                                      topk_metric)
                        if code_vectors_file is not None:
                            self._export_code_vectors(code_vectors_file, text, code_vectors)
                    if total_batches % cfg.NUM_BATCHES_TO_LOG_PROGRESS == 0:
                        self._trace_evaluation(total_predictions, time.time() - start_time)
                self.log("Done evaluating, epoch reached")
                if writer:
                    topk_metric.nr_correct_predictions = topk_metric.nr_correct_predictions + np.cumsum(hist).astype(np.float64)
                    topk_metric.nr_predictions += int(counts[0])
                    subtokens_metric.nr_predictions += int(counts[0])
                    subtokens_metric.nr_true_positives += int(counts[1])
                    subtokens_metric.nr_false_positives += int(counts[2])
                    subtokens_metric.nr_false_negatives += int(counts[3])
                    log_output_file.write(str(topk_metric.topk_correct_predictions) + "\n")
        except BaseException:
            reader.close()                         # a pass that stopped early leaves rows queued: the next is a new reader
            self._dev_eval_reader = None
            raise
        finally:
            if code_vectors_file is not None:
                self._close_code_vectors(code_vectors_file, text)
        self.log("Device evaluation: %.1f MB of text uploaded, %.1f MB of device memory held" % (
            reader.h2d_bytes / 1e6, reader.device_bytes() / 1e6))
        elapsed = int(time.time() - eval_start_time)
        self.log("Evaluation time: %sH:%sM:%sS" % ((elapsed // 60 // 60), (elapsed // 60) % 60, elapsed % 60))
        results = None
        if writer:
            results = ModelEvaluationResults(topk_acc=topk_metric.topk_correct_predictions,
                                             subtoken_precision=subtokens_metric.precision,
                                             subtoken_recall=subtokens_metric.recall, subtoken_f1=subtokens_metric.f1)
        if self.world > 1:                         # every rank returns rank 0's results
            import torch.distributed as dist
            gathered = [None] * self.world
            dist.all_gather_object(gathered, results)
            results = gathered[0]
        return results

    # ---- `.vectors` and word2vec files (C2V_DEVICE_TEXT=1 formats them on the GPU, DESIGN.md §6f) ----------------------
    def _open_code_vectors(self, writer: bool):
        """(`<test file>.vectors` opened for this evaluation, or None when it exports none or is not the writing rank;
        with C2V_DEVICE_TEXT=1 the DeviceTextWriter that fills it, else None)."""
        cfg = self.config
        if not (cfg.EXPORT_CODE_VECTORS and writer):
            return None, None
        if not self._device_text:
            return open(cfg.TEST_DATA_PATH + ".vectors", "w"), None
        f = open(cfg.TEST_DATA_PATH + ".vectors", "wb")
        return f, DeviceTextWriter(f, self.engine.dev)

    def _export_code_vectors(self, file, text: Optional[DeviceTextWriter], code_vectors):
        """One batch's lines of the `.vectors` file: _write_code_vectors, or formatted on the GPU from the device tensor
        (a host array is uploaded again)."""
        if text is None:
            self._write_code_vectors(file, code_vectors)
            return
        import torch
        text.write_rows(code_vectors if isinstance(code_vectors, torch.Tensor) else
                        self.engine.to_device(code_vectors, torch.float32))

    def _close_code_vectors(self, file, text: Optional[DeviceTextWriter]):
        try:
            if text is not None:
                text.close()
                self.log("Device text: %s" % text.report())
        finally:
            file.close()

    def _log_and_score_host_rows(self, sc, n: int, index_to_word, output_file, subtokens_metric, topk_metric):
        """log.txt lines of one scored batch, in row order: the three line forms of _log_predictions_during_evaluation
        from the kernel's rank and first legal word, and for flagged rows that method itself; the flagged rows then go
        through the host metrics (SubtokensEvaluationMetric raises IndexError for a top-k without a legal word)."""
        names, off = sc.names
        lines, host_rows = [], []
        for j in range(n):
            name = names[off[j]:off[j + 1]].decode("utf-8")
            if sc.flags[j]:
                top_words = self.vocabs.target_vocab.lookup_word(sc.ids[j])
                output_file.write("".join(lines))
                lines = []
                self._log_predictions_during_evaluation([(name, top_words)], output_file)
                host_rows.append((name, top_words))
                continue
            r = int(sc.rank[j])
            if r < 0:
                lines.append("No results for predicting: " + name)
            elif r == 0:
                lines.append("Original: " + name + ", predicted 1st: " + index_to_word[int(sc.first[j])] + "\n")
            else:
                lines.append("\t\t predicted correctly at rank: " + str(r + 1) + "\n")
        output_file.write("".join(lines))
        if host_rows:
            topk_metric.update_batch(host_rows)
            subtokens_metric.update_batch(host_rows)

    def _predict_sharded_device(self, tensors, n_all: int, want_code: bool):
        """_predict_sharded on a batch already in device memory: (top-k ids [n, k], code vectors [n, D] or None) as
        device tensors, the slices and padding as there, the ids all-gathered into device memory."""
        import torch
        import torch.distributed as dist
        e, W, r = self.engine, self.world, self.rank
        idx_parts, code_parts = [], []
        for s in range(0, n_all, W * e.local_batch):
            n = min(W * e.local_batch, n_all - s)
            b = -(-n // W)
            rows = torch.clamp(torch.arange(s + r * b, s + (r + 1) * b, device=e.dev), max=s + n - 1)
            idx, _val, code = self.trainer.predict(*(t.index_select(0, rows) for t in tensors), normalize=0)
            idx_all = torch.empty((W * b, idx.shape[1]), dtype=idx.dtype, device=e.dev)
            dist.all_gather_into_tensor(idx_all, idx)
            idx_parts.append(idx_all[:n])
            if want_code:
                code_all = torch.empty((W * b, code.shape[1]), dtype=code.dtype, device=e.dev)
                dist.all_gather_into_tensor(code_all, code)
                code_parts.append(code_all[:n])
        return torch.cat(idx_parts).contiguous(), (torch.cat(code_parts) if want_code else None)

    def _predict_sharded(self, t: ReaderInputTensors, want_code: bool):
        """(top-k ids [n, k], code vectors [n, D] or None) of the n rows of one reader batch, on rank 0; the other ranks
        get the same arrays.  The rows go in global batches of at most world * local_batch rows: each rank takes an
        equal slice (the last global batch padded with copies of its last row), Trainer.predict ranks it against the
        whole target table, and the slices are all-gathered back in file order without the padding."""
        import torch
        import torch.distributed as dist
        e, W, r = self.engine, self.world, self.rank
        arrays = ((t.path_source_token_indices, torch.int32), (t.path_indices, torch.int32),
                  (t.path_target_token_indices, torch.int32), (t.context_valid_mask, torch.float32))
        n_all = int(t.path_source_token_indices.shape[0])
        idx_parts, code_parts = [], []
        for s in range(0, n_all, W * e.local_batch):
            n = min(W * e.local_batch, n_all - s)
            b = -(-n // W)
            rows = np.minimum(np.arange(s + r * b, s + (r + 1) * b), s + n - 1)
            idx, _val, code = self.trainer.predict(*(e.to_device(a[rows], dt) for a, dt in arrays), normalize=0)
            idx_all = torch.empty((W * b, idx.shape[1]), dtype=idx.dtype, device=e.dev)
            dist.all_gather_into_tensor(idx_all, idx)
            idx_parts.append(idx_all[:n].cpu().numpy())
            if want_code:
                code_all = torch.empty((W * b, code.shape[1]), dtype=code.dtype, device=e.dev)
                dist.all_gather_into_tensor(code_all, code)
                code_parts.append(code_all[:n].cpu().numpy())
        return np.concatenate(idx_parts), (np.concatenate(code_parts) if want_code else None)

    # ---- predict (tensorflow_model.py:311-368) ----------------------------------------------------------
    def predict(self, predict_data_lines: Iterable[str]) -> List[ModelPredictionResults]:
        if self.predict_reader is None:
            self.predict_reader = PathContextReader(vocabs=self.vocabs, model_input_tensors_former=_EvaluateInputFormer(),
                                                    config=self.config, estimator_action=EstimatorAction.Predict)
        results: List[ModelPredictionResults] = []
        self.engine.set_option("math_mode", self._math_eval)
        for line in predict_data_lines:
            t = _EvaluateInputFormer().from_model_input_form(self.predict_reader.process_input_row(line))
            idx, scores, code_vectors, attn = self.engine.predict_batch_host(
                t.path_source_token_indices, t.path_indices, t.path_target_token_indices, t.context_valid_mask,
                normalize=True, want_code=True, want_attention=True)
            assert idx.shape[0] == 1
            top_words = self.vocabs.target_vocab.lookup_word(idx[0])
            attention_per_context = self._get_attention_weight_per_context(
                t.path_source_token_strings[0], t.path_strings[0], t.path_target_token_strings[0], attn[0])
            results.append(ModelPredictionResults(
                original_name=common.binary_to_string(t.target_string[0]), topk_predicted_words=top_words,
                topk_predicted_words_scores=scores[0], attention_per_context=attention_per_context,
                code_vector=(code_vectors[0] if self.config.EXPORT_CODE_VECTORS else None)))
        return results

    # ---- `--predict` on the GPU (C2V_DEVICE_PREDICT=1, DESIGN.md §6i) ------------------------------------------------
    _PREDICT_NORMALIZE = 1                     # softmax over the k scores, as predict() asks the engine for

    @property
    def device_predict(self) -> bool:
        return self._device_predict

    def print_predictions_device(self, data: bytes, universal_newlines: bool, out) -> bool:
        """__main__.print_predictions over the extractor output `data` (a file read in text mode when
        universal_newlines, else standard input), predicted and formatted on the GPU and written to the binary stream
        `out`, byte for byte the host route's text.  False, with nothing written, for an input that needs the host route
        (a byte >= 0x80, or a path the device's key table cannot hold: device_predict.py)."""
        from .device_predict import DevicePredictor
        if self.world > 1:
            raise ValueError("--predict runs on one GPU; this run has %d ranks" % self.world)
        if self._dev_predictor is None:
            self._dev_predictor = DevicePredictor(self, self._PREDICT_NORMALIZE)
        p = self._dev_predictor
        done = p.run(data, universal_newlines, out, want_code=self.config.EXPORT_CODE_VECTORS)
        if not done:
            self.log("Device predict: the input needs the host route (a byte >= 0x80, a numeric path that is not the "
                     "decimal of an int32, or a path of 1 MB or more); predicting it one method at a time on the host")
        else:
            self.log("Device predict: %.1f MB of device memory held, %.1f MB page-locked" % (
                p.device_bytes() / 1e6, p.pinned_bytes / 1e6))
        return done

    def _get_vocab_embedding_as_np_array(self, vocab_type: VocabType) -> np.ndarray:
        assert vocab_type in VocabType
        return self._vocab_embedding_on_device(vocab_type).cpu().numpy()

    def _vocab_embedding_on_device(self, vocab_type: VocabType):
        """The whole table of `vocab_type` as a device tensor; on several GPUs gathered on every rank (a collective)."""
        if self.world > 1:
            return self._gather_table(self._param_of_vocab[vocab_type])
        self.engine.sync_tables()
        return self.engine.params[self._param_of_vocab[vocab_type]].detach()

    # ---- nearest neighbours (similarity.py, DESIGN.md §6h) ------------------------------------------------------------
    def _knn(self):
        """The model's search handle, made once (one GPU only, as --predict)."""
        from .similarity import NearestNeighbours
        if self.world > 1:
            raise ValueError("most_similar and nearest_code_vectors run on one GPU; this run has %d ranks" % self.world)
        if getattr(self, "_knn_handle", None) is None:
            self._knn_handle = NearestNeighbours(self.engine.dev)
            self._knn_bound = None
        return self._knn_handle

    def most_similar(self, positive, negative=(), topn: int = 10, vocab_type: VocabType = VocabType.Target):
        """gensim 4's KeyedVectors.most_similar(positive, negative, topn) on the table of `vocab_type`, on the GPU:
        [(word, cosine similarity)], the query's own words left out.  KeyError for a word outside the vocabulary."""
        from . import similarity
        if isinstance(positive, str):
            positive = [positive]
        if isinstance(negative, str):
            negative = [negative]
        nn = self._knn()
        vocab = self.vocabs.get(vocab_type)
        for w in list(positive) + list(negative):
            if w not in vocab.word_to_index:
                raise KeyError("Key '%s' not present in vocabulary" % w)
        # the table as it stands after the engine's last step: re-bound whenever a step has run since
        stamp = (vocab_type, self._math_eval, self.engine.launch_count)
        if self._knn_bound != stamp:
            nn.bind(self._vocab_embedding_on_device(vocab_type), self._math_eval)
            self._knn_bound = (vocab_type, self._math_eval, self.engine.launch_count)
        return similarity.most_similar(nn, vocab.word_to_index, vocab.index_to_word, positive, negative, topn)

    def nearest_code_vectors(self, c2v_path: str, topn: int = 10):
        """The code vectors of the examples of `c2v_path` that evaluate() scores -- in its order and its batches of
        TEST_BATCH_SIZE, equal to what --export_code_vectors writes -- and each one's topn nearest other examples by
        cosine: (names [N], code vectors [N, D] on the host, neighbour rows [N, topn], similarities [N, topn]), rows
        padded with (INT_MAX, -inf) when the corpus has fewer than topn + 1 examples."""
        import copy
        import torch
        from . import similarity
        if self._device_eval:
            return self._nearest_device(c2v_path, topn)
        nn = self._knn()
        cfg = copy.copy(self.config)
        cfg.TEST_DATA_PATH = c2v_path
        reader = PathContextReader(vocabs=self.vocabs, model_input_tensors_former=_EvaluateInputFormer(), config=cfg,
                                   estimator_action=EstimatorAction.Evaluate)
        self.engine.set_option("math_mode", self._math_eval)
        names, parts = [], []
        for batch in reader.get_dataset():
            t = _EvaluateInputFormer().from_model_input_form(batch)
            _idx, _vals, code, _attn = self.engine.predict_batch_host(
                t.path_source_token_indices, t.path_indices, t.path_target_token_indices, t.context_valid_mask,
                normalize=False, want_code=True, want_attention=False)
            names.extend(common.binary_to_string(n) for n in t.target_string)
            parts.append(code)
        D = self.config.CODE_VECTOR_SIZE
        vectors = np.concatenate(parts) if parts else np.zeros((0, D), dtype=np.float32)
        if vectors.shape[0] == 0:
            return names, vectors, np.zeros((0, topn), np.int32), np.zeros((0, topn), np.float32)
        self._knn_bound = None
        idx, val = similarity.nearest_rows(nn, torch.from_numpy(vectors).to(self.engine.dev), topn, self._math_eval)
        self.log("Nearest neighbours: %d code vectors, %.1f MB of device memory held" % (
            vectors.shape[0], nn.device_bytes() / 1e6))
        return names, vectors, idx, val

    # ---- name scores (name_scores.py, DESIGN.md §6n) ------------------------------------------------------------------
    def score_names(self, c2v_path: str):
        """The examples of `c2v_path` that evaluate() scores -- in its order and its batches of TEST_BATCH_SIZE -- with each
        one's own name scored over the whole target vocabulary on the GPU (c2v_name_scores): (names [N], target ids [N],
        rank [N], logp [N], top1 [N], top1_logp [N]) as host arrays.  A name outside the target vocabulary has the OOV
        word's id, and its rank and logp are that word's.  The full-softmax quantities are the same for both frameworks."""
        import copy
        import torch
        if self.world > 1:
            raise ValueError("score_names runs on one GPU; this run has %d ranks" % self.world)
        if self._device_eval:
            return self._score_names_device(c2v_path)
        cfg = copy.copy(self.config)
        cfg.TEST_DATA_PATH = c2v_path
        reader = PathContextReader(vocabs=self.vocabs, model_input_tensors_former=_EvaluateInputFormer(), config=cfg,
                                   estimator_action=EstimatorAction.Evaluate)
        e = self.engine
        e.set_option("math_mode", self._math_eval)
        names, parts = [], []
        for batch in reader.get_dataset():
            t = _EvaluateInputFormer().from_model_input_form(batch)
            batch_names = [common.binary_to_string(n) for n in t.target_string]
            ids = self.vocabs.target_vocab.lookup_index(batch_names)
            code, _ = e.forward(e.to_device(t.path_source_token_indices, torch.int32), e.to_device(t.path_indices, torch.int32),
                                e.to_device(t.path_target_token_indices, torch.int32),
                                e.to_device(t.context_valid_mask, torch.float32), want_attention=False)
            scores = e.name_scores(code, e.to_device(ids, torch.int32))
            parts.append([ids] + [x.cpu().numpy() for x in scores])
            names.extend(batch_names)
        if not parts:
            return (names, *(np.zeros(0, dt) for dt in (np.int32, np.int32, np.float32, np.int32, np.float32)))
        return (names, *(np.concatenate(c) for c in zip(*parts)))

    # ---- --score_names and --nearest on the GPU (C2V_DEVICE_EVAL=1, DESIGN.md §6o) -----------------------------------
    @property
    def device_eval(self) -> bool:
        return self._device_eval

    def _device_corpus_reader(self, c2v_path: str):
        """The GPU evaluation reader of the corpus `c2v_path` (not TEST_DATA_PATH), sharing the model's device
        vocabularies; made once per path (and again after a pass that failed).  Its names are checked as UTF-8 chunk by
        chunk, as the host reader decodes them."""
        import copy
        from .device_reader import DeviceBatchReader, eval_tables
        if self._dev_corpus_reader is not None and self._dev_corpus_path != c2v_path:
            self._dev_corpus_reader.close()
            self._dev_corpus_reader = None
        if self._dev_corpus_reader is None:
            cfg = copy.copy(self.config)
            cfg.TEST_DATA_PATH = c2v_path
            reader = PathContextReader(vocabs=self.vocabs, model_input_tensors_former=_EvaluateInputFormer(), config=cfg,
                                       estimator_action=EstimatorAction.Evaluate)
            if self._eval_tables is None:
                self._eval_tables = eval_tables(self.vocabs.target_vocab)
            self._dev_corpus_reader = DeviceBatchReader(reader, self.engine.dev, vocabs=self._shared_device_vocabs(reader),
                                                        tables=self._eval_tables, check_utf8=True)
            self._dev_corpus_path = c2v_path
        return self._dev_corpus_reader

    def _device_corpus_pass(self, c2v_path: str, per_batch):
        """One pass over the examples of `c2v_path` that evaluate() scores, in its order and its batches of
        TEST_BATCH_SIZE, read and encoded on the GPU: per_batch(batch, n, code) for each batch of n rows, with its code
        vectors [n, D] (device) in the evaluation math mode.  per_batch queues its device work on the current stream
        (the batch's slot is handed back after it).  The host reader's exceptions for a malformed corpus are raised."""
        if self.world > 1:
            raise ValueError("--score_names and --nearest run on one GPU; this run has %d ranks" % self.world)
        reader = self._device_corpus_reader(c2v_path)
        e = self.engine
        e.set_option("math_mode", self._math_eval)
        try:
            for batch in reader:
                batch.wait()
                n = batch.hi - batch.lo
                code, _ = e.forward(*batch.tensors[:4], want_attention=False)
                per_batch(batch, n, code)
                batch.release()
        except BaseException:
            reader.close()                             # a pass that stopped early leaves rows queued
            self._dev_corpus_reader = None
            raise

    @staticmethod
    def _host_names(names, off, n: int) -> List[str]:
        """The n names names[off[j], off[j + 1]) (device uint8 / int64) decoded on the host."""
        off = off[:n + 1].cpu().numpy()
        blob = names[:int(off[n])].cpu().numpy().tobytes()
        return [blob[off[j]:off[j + 1]].decode("utf-8") for j in range(n)]

    def _score_names_device(self, c2v_path: str, stage=None):
        """score_names on the GPU route: the same arrays.  With a corpus_text.LineStage, each batch's lines of
        `<corpus>.name_scores` are formatted on the GPU into it, and the names stay on the device (None is returned for
        them)."""
        import ctypes as C
        e, lib = self.engine, self.engine.lib
        vocab = self.vocabs.target_vocab
        oov = vocab.word_to_index[vocab.special_words.OOV]
        names, parts = ([] if stage is None else None), []

        def per_batch(batch, n, code):
            target = batch.tensors[4]
            rank, logp, top1, top1_logp = e.name_scores(code, target)
            s = batch._slot
            if stage is not None:
                words, word_off, n_words = self._dev_corpus_reader.eval_words()
                scratch, scratch_bytes = stage.scratch_for(n)

                def fmt(out, cap, total):
                    e._check(lib.c2v_name_scores_text(
                        n, s["names"].data_ptr(), s["name_off"].data_ptr(), target.data_ptr(), oov, rank.data_ptr(),
                        logp.data_ptr(), top1.data_ptr(), top1_logp.data_ptr(), words, word_off, n_words, scratch,
                        scratch_bytes, out, cap, total, e._stream()))
                stage.emit(fmt)
            else:
                names.extend(self._host_names(s["names"], s["name_off"], n))
            parts.append([x.cpu().numpy() for x in (target, rank, logp, top1, top1_logp)])

        self._device_corpus_pass(c2v_path, per_batch)
        if not parts:
            return (names, *(np.zeros(0, dt) for dt in (np.int32, np.int32, np.float32, np.int32, np.float32)))
        return (names, *(np.concatenate(c) for c in zip(*parts)))

    def write_name_scores_device(self, c2v_path: str) -> str:
        """`<c2v_path>.name_scores` read, scored and formatted on the GPU: __main__.write_name_scores' bytes and summary
        line.  The file appears only once the whole corpus is scored (a corpus the reader rejects leaves none)."""
        from . import name_scores
        from .corpus_text import LineStage, atomic_output
        out_path = c2v_path + name_scores.SUFFIX
        with atomic_output(out_path) as f:
            stage = LineStage(f, self.engine.dev)
            try:
                _, target, rank, logp, _, _ = self._score_names_device(c2v_path, stage)
            finally:
                stage.close()
        self.corpus_text_stage = stage             # its timings and peak memory (tools/corpus_rate.py)
        vocab = self.vocabs.target_vocab
        in_vocab = target != vocab.word_to_index[vocab.special_words.OOV]
        self.log(name_scores.summary_line(rank, logp, in_vocab))
        return out_path

    def _nearest_device(self, c2v_path: str, topn: int, stage=None):
        """nearest_code_vectors on the GPU route: the code vectors [N, D] and the names of the N rows gathered in device
        memory, then c2v_knn_search.  Without a stage, the host arrays nearest_code_vectors returns; with a
        corpus_text.LineStage, the lines of `<corpus>.nearest` formatted on the GPU into it, and None."""
        import torch
        from . import similarity
        from .corpus_text import NEAREST_ROWS
        nn = self._knn()
        e = self.engine
        D = self.config.CODE_VECTOR_SIZE
        acc = {"n": 0, "vec": None, "names": None, "off": None, "name_bytes": 0}
        nb_host = torch.zeros(1, dtype=torch.int64).pin_memory()

        def grow(t, need, make):
            if t is not None and t.shape[0] >= need:
                return t
            bigger = make(max(need, 2 * (0 if t is None else t.shape[0]), 1024))
            if t is not None:
                bigger[:t.shape[0]].copy_(t)
            return bigger

        def per_batch(batch, n, code):
            s = batch._slot
            nb_host.copy_(s["name_off"][n:n + 1])                     # the batch's name bytes
            N, base = acc["n"], acc["name_bytes"]
            acc["vec"] = grow(acc["vec"], N + n, lambda m: torch.empty((m, D), dtype=torch.float32, device=e.dev))
            acc["off"] = grow(acc["off"], N + n + 1, lambda m: torch.zeros(m, dtype=torch.int64, device=e.dev))
            acc["vec"][N:N + n].copy_(code)
            acc["off"][N + 1:N + n + 1].copy_(s["name_off"][1:n + 1] + base)
            nb = int(nb_host[0])
            acc["names"] = grow(acc["names"], base + nb, lambda m: torch.empty(m, dtype=torch.uint8, device=e.dev))
            acc["names"][base:base + nb].copy_(s["names"][:nb])
            acc["n"], acc["name_bytes"] = N + n, base + nb

        self._device_corpus_pass(c2v_path, per_batch)
        N = acc["n"]
        if N == 0:
            empty = (np.zeros((0, D), dtype=np.float32), np.zeros((0, topn), np.int32), np.zeros((0, topn), np.float32))
            return None if stage is not None else ([], *empty)
        vectors = acc["vec"][:N]
        self._knn_bound = None
        idx, val = similarity.nearest_rows_device(nn, vectors, topn, self._math_eval)
        self.log("Nearest neighbours: %d code vectors, %.1f MB of device memory held" % (N, nn.device_bytes() / 1e6))
        if stage is None:
            names = self._host_names(acc["names"], acc["off"], N)
            return names, vectors.cpu().numpy(), idx.cpu().numpy(), val.cpu().numpy()
        for r0 in range(0, N, NEAREST_ROWS):
            n = min(NEAREST_ROWS, N - r0)
            scratch, scratch_bytes = stage.scratch_for(n)

            def fmt(out, cap, total, r0=r0, n=n):
                e._check(e.lib.c2v_nearest_text(r0, n, N, topn, acc["names"].data_ptr(), acc["off"].data_ptr(),
                                                idx.data_ptr(), val.data_ptr(), scratch, scratch_bytes, out, cap, total,
                                                e._stream()))
            stage.emit(fmt)
        return None

    def write_nearest_device(self, c2v_path: str, topn: int) -> str:
        """`<c2v_path>.nearest` read, searched and formatted on the GPU: __main__.write_nearest's bytes, without the
        [N, D] code vectors leaving the device.  The file appears only once the whole corpus is searched."""
        from .corpus_text import LineStage, atomic_output
        out_path = c2v_path + ".nearest"
        with atomic_output(out_path) as f:
            stage = LineStage(f, self.engine.dev)
            try:
                self._nearest_device(c2v_path, topn, stage)
            finally:
                stage.close()
        self.corpus_text_stage = stage             # its timings and peak memory (tools/corpus_rate.py)
        return out_path

    def _gather_table(self, name: str):
        """The whole table `name` on every rank (a collective), in device memory: the embedding shards all-gathered and
        interleaved back (global row = local row * world + rank), or the target blocks all-gathered and concatenated."""
        import torch
        import torch.distributed as dist
        e, W = self.engine, self.world
        if name in ("tok", "path"):
            shard = e.shard_params[name]
            whole = torch.empty((W,) + tuple(shard.shape), dtype=shard.dtype, device=e.dev)
            dist.all_gather_into_tensor(whole, shard)
            n_rows = self._engine_dims().shapes()[name][0]
            return whole.transpose(0, 1).reshape(-1, shard.shape[1])[:n_rows]
        Y, per = e.global_target_vocab, -(-e.global_target_vocab // W)     # blocks of `per` rows, the last one shorter
        block = torch.zeros((per, e.dims.code_dim), dtype=torch.float32, device=e.dev)
        block[:e.dims.target_vocab].copy_(e.params["tgt"])
        whole = torch.empty((W * per, e.dims.code_dim), dtype=torch.float32, device=e.dev)
        dist.all_gather_into_tensor(whole, block)
        return whole[:Y]

    def save_word2vec_format(self, dest_save_path: str, vocab_type: VocabType):
        if self.world > 1 and self.rank != 0:
            self._vocab_embedding_on_device(vocab_type)              # the gather is a collective; rank 0 writes the file
            return
        if not self._device_text:
            return super().save_word2vec_format(dest_save_path, vocab_type)
        if vocab_type not in VocabType:
            raise ValueError("`vocab_type` should be `VocabType.Token`, `VocabType.Target` or `VocabType.Path`.")
        from . import text_export
        vocab = self.vocabs.get(vocab_type)
        table = self._vocab_embedding_on_device(vocab_type)
        with open(dest_save_path, "w") as out:
            text = text_export.save_word2vec_file(out, vocab.index_to_word, table)
        self.log("Device text: %s" % text.report())

    # ---- logging helpers (tensorflow_model.py:411-437) ------------------------------------------------------
    def _log_predictions_during_evaluation(self, results, output_file):
        special = self.vocabs.target_vocab.special_words
        for original_name, top_predicted_words in results:
            found = common.get_first_match_word_from_top_predictions(special, original_name, top_predicted_words)
            if found is None:
                output_file.write("No results for predicting: " + original_name)
                continue
            rank, word = found
            if rank == 0:
                output_file.write("Original: " + original_name + ", predicted 1st: " + word + "\n")
            else:
                output_file.write("\t\t predicted correctly at rank: " + str(rank + 1) + "\n")

    def _trace_training(self, sum_loss, batch_num, multi_batch_start_time):
        cfg = self.config
        elapsed = time.time() - multi_batch_start_time
        # the reference divides the summed mean losses by NUM_BATCHES * BATCH_SIZE (:426); kept as is
        avg_loss = sum_loss / (cfg.NUM_BATCHES_TO_LOG_PROGRESS * cfg.TRAIN_BATCH_SIZE)
        throughput = cfg.TRAIN_BATCH_SIZE * cfg.NUM_BATCHES_TO_LOG_PROGRESS / (elapsed if elapsed > 0 else 1)
        self.log("Average loss at batch %d: %f, \tthroughput: %d samples/sec" % (batch_num, avg_loss, throughput))

    def _trace_evaluation(self, total_predictions, elapsed):
        self.log("Evaluated %d examples..." % total_predictions)
        self.log("Prediction throughput: %d samples/sec" % int(total_predictions / (elapsed if elapsed > 0 else 1)))


# ---- host-side metrics (tensorflow_model.py:450-516) ---------------------------------------------------
class SubtokensEvaluationMetric:
    def __init__(self, filter_impossible_names_fn):
        self.nr_true_positives = 0
        self.nr_false_positives = 0
        self.nr_false_negatives = 0
        self.nr_predictions = 0
        self.filter_impossible_names_fn = filter_impossible_names_fn

    def update_batch(self, results):
        for original_name, top_words in results:
            prediction = self.filter_impossible_names_fn(top_words)[0]      # IndexError if none is legal, as upstream
            truth = Counter(common.get_subtokens(original_name))
            guess = Counter(common.get_subtokens(prediction))
            self.nr_true_positives += sum(n for tok, n in guess.items() if tok in truth)
            self.nr_false_positives += sum(n for tok, n in guess.items() if tok not in truth)
            self.nr_false_negatives += sum(n for tok, n in truth.items() if tok not in guess)
            self.nr_predictions += 1

    @property
    def true_positive(self):
        return self.nr_true_positives / self.nr_predictions

    @property
    def false_positive(self):
        return self.nr_false_positives / self.nr_predictions

    @property
    def false_negative(self):
        return self.nr_false_negatives / self.nr_predictions

    @property
    def precision(self):
        return self.nr_true_positives / (self.nr_true_positives + self.nr_false_positives)

    @property
    def recall(self):
        return self.nr_true_positives / (self.nr_true_positives + self.nr_false_negatives)

    @property
    def f1(self):
        p, r = self.precision, self.recall
        return 0 if p + r == 0 else 2 * p * r / (p + r)


class TopKAccuracyEvaluationMetric:
    def __init__(self, top_k: int, get_first_match_word_from_top_predictions_fn):
        self.top_k = top_k
        self.nr_correct_predictions = np.zeros(self.top_k)
        self.nr_predictions = 0
        self.get_first_match_word_from_top_predictions_fn = get_first_match_word_from_top_predictions_fn

    def update_batch(self, results):
        for original_name, top_predicted_words in results:
            self.nr_predictions += 1
            found = self.get_first_match_word_from_top_predictions_fn(original_name, top_predicted_words)
            if found is not None:
                self.nr_correct_predictions[found[0]:self.top_k] += 1

    @property
    def topk_correct_predictions(self):
        return self.nr_correct_predictions / self.nr_predictions


# ---- tuple orders the model consumes (tensorflow_model.py:519-551) ---------------------------------------
class _TrainInputFormer(ModelInputTensorsFormer):
    def to_model_input_form(self, t: ReaderInputTensors):
        return (t.target_index, t.path_source_token_indices, t.path_indices, t.path_target_token_indices,
                t.context_valid_mask)

    def from_model_input_form(self, row) -> ReaderInputTensors:
        return ReaderInputTensors(target_index=row[0], path_source_token_indices=row[1], path_indices=row[2],
                                  path_target_token_indices=row[3], context_valid_mask=row[4])


class _EvaluateInputFormer(ModelInputTensorsFormer):
    def to_model_input_form(self, t: ReaderInputTensors):
        return (t.target_string, t.path_source_token_indices, t.path_indices, t.path_target_token_indices,
                t.context_valid_mask, t.path_source_token_strings, t.path_strings, t.path_target_token_strings)

    def from_model_input_form(self, row) -> ReaderInputTensors:
        return ReaderInputTensors(target_string=row[0], path_source_token_indices=row[1], path_indices=row[2],
                                  path_target_token_indices=row[3], context_valid_mask=row[4],
                                  path_source_token_strings=row[5], path_strings=row[6],
                                  path_target_token_strings=row[7])
