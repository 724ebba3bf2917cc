"""`Code2VecModel` for `--framework b200-keras`: the engine behind the reference's *Keras* backend.

The Keras backend (keras_model.py:27-316) is the same architecture as the TensorFlow one with
different numerics and bookkeeping (SURVEY A.4).  What changes relative to `b200_model`:

  initialisers   `Embedding` layers and the attention vector U(+-0.05); both Dense kernels
                 glorot-uniform -- the output kernel is [D, |Y|] in Keras and is held here row-major
                 as [|Y|, D] (keras_model.py:46-70, keras_attention_layer.py:29-34, :310-316)
  optimizer      `tf.optimizers.Adam()`: epsilon 1e-7 instead of 1e-8 (keras_model.py:115-117);
                 the sparse (embedding) update is dense/non-lazy there as well
  loss           'sparse_categorical_crossentropy' on the softmax output (keras_model.py:128-130):
                 Keras recovers the logits of a Softmax op and calls the fused
                 softmax-cross-entropy [TF-lib], i.e. the same value as the TF backend's loss
  scores         top-k over the softmax of the WHOLE target vocabulary, scores = those
                 probabilities (keras_topk_word_predictions_layer.py:30-35) -- `normalize=2`
  evaluate()     per-k `sparse_top_k_categorical_accuracy` on the target INDEX (no legality
                 filter), subtoken precision/recall/F1 with the first legal word of the top-k, and
                 the mean loss (keras_model.py:96-113,181-194)
  train()        `fit` cadence: epochs x steps_per_epoch, progress every NUM_BATCHES_TO_LOG_PROGRESS,
                 evaluation every NUM_TRAIN_BATCHES_TO_EVALUATE batches and at each epoch end, a
                 checkpoint every SAVE_EVERY_EPOCHS epochs (keras_model.py:147-179,320-371;
                 keras_checkpoint_saver_callback.py:29-129)
The arithmetic is the same C-ABI engine; nothing here touches TensorFlow.
"""
from __future__ import annotations

import datetime
import re
import time
from typing import Iterable, List, Optional

import numpy as np

from .b200_model import Code2VecModel as _TFNumericsModel
from .b200_model import _EvaluateInputFormer, _TrainInputFormer, _prefetch, _with_next
from .common import common
from .model_base import ModelEvaluationResults, ModelPredictionResults
from .path_context_reader import EstimatorAction, ModelInputTensorsFormer, PathContextReader, ReaderInputTensors

KERAS_ADAM = dict(lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-7)      # tf.optimizers.Adam() defaults [TF-lib]
_LEGAL_WORD = re.compile(r"^[a-zA-Z\|]+$")                         # keras_model.py:104


class _KerasEvaluateInputFormer(ModelInputTensorsFormer):
    """Evaluate rows carry both the target index (loss, top-k accuracy) and its string (subtoken
    metrics) -- the `targets` dict of keras_model.py:388-391."""

    def to_model_input_form(self, t: ReaderInputTensors):
        return (t.path_source_token_indices, t.path_indices, t.path_target_token_indices, t.context_valid_mask,
                t.target_index, t.target_string)

    def from_model_input_form(self, row) -> ReaderInputTensors:
        return ReaderInputTensors(path_source_token_indices=row[0], path_indices=row[1], path_target_token_indices=row[2],
                                  context_valid_mask=row[3], target_index=row[4], target_string=row[5])


class SubtokenCounts:
    """tp / fp / fn of WordsSubtokenMetricBase.update_state (keras_words_subtoken_metrics.py:35-86):
    every predicted subtoken found in the true name is a true positive, every other one a false
    positive, every true subtoken missing from the prediction a false negative (duplicates count)."""

    def __init__(self):
        self.tp = self.fp = self.fn = 0.0

    def update(self, true_word: str, predicted_word: str):
        truth, guess = true_word.split("|"), predicted_word.split("|")
        self.tp += sum(1 for s in guess if s in truth)
        self.fp += sum(1 for s in guess if s not in truth)
        self.fn += sum(1 for s in truth if s not in guess)

    @staticmethod
    def _div(a, b):
        return a / b if b else 0.0                              # tf.math.divide_no_nan

    @property
    def precision(self):
        return self._div(self.tp, self.tp + self.fp)

    @property
    def recall(self):
        return self._div(self.tp, self.tp + self.fn)

    @property
    def f1(self):
        p, r = self.precision, self.recall
        return self._div(2 * p * r, p + r + 1e-7)               # K.epsilon() in the denominator (:137)


class Code2VecModel(_TFNumericsModel):
    _ADAM = KERAS_ADAM
    _INIT_SCHEME = "keras"

    def __init__(self, config):
        self.nr_epochs_trained = 0                              # ModelTrainingStatus (keras_checkpoint_saver_callback.py:14-17)
        self._avg_eval_duration: Optional[float] = None
        super().__init__(config)

    # ---- engine life cycle -------------------------------------------------------------------
    def _create_inner_model(self):
        self._make_engine()
        self.engine.init_params(scheme="keras")
        for name, shape in self.engine.dims.shapes().items():
            self.log("variable name: {} -- shape: {} -- #params: {}".format(name, shape, int(np.prod(shape))))

    # ---- train: the schedule `keras_train_model.fit` + callbacks produce ---------------------------
    def train(self):
        cfg = self.config
        self.log("Starting training...")
        reader = PathContextReader(vocabs=self.vocabs, model_input_tensors_former=_TrainInputFormer(), config=cfg,
                                   estimator_action=EstimatorAction.Train, repeat_endlessly=True, shuffle_seed=self._seed)
        batches = _with_next(_prefetch(reader.get_dataset()))
        former = _TrainInputFormer()
        steps = cfg.train_steps_per_epoch
        last_saved_epoch = self.nr_epochs_trained
        avg_throughput = None
        self.engine.set_option("math_mode", self._math_train)
        for epoch in range(self.nr_epochs_trained, cfg.NUM_TRAIN_EPOCHS):
            window_loss, window_start, epoch_loss = 0.0, time.time(), 0.0
            for batch_idx in range(steps):
                try:
                    batch, following = next(batches)
                except StopIteration:
                    break
                t = former.from_model_input_form(batch)
                n = former.from_model_input_form(following) if (self._hint_next and following is not None) else None
                self.engine.set_option("math_mode", self._math_train)
                loss = self.trainer.step_host(
                    t.path_source_token_indices, t.path_indices, t.path_target_token_indices, t.context_valid_mask, t.target_index,
                    next_batch=None if n is None else (n.path_source_token_indices, n.path_indices, n.path_target_token_indices))
                window_loss += loss
                epoch_loss += loss
                done = batch_idx + 1
                if done % cfg.NUM_BATCHES_TO_LOG_PROGRESS == 0:
                    elapsed = max(time.time() - window_start, 1e-9)
                    throughput = cfg.TRAIN_BATCH_SIZE * cfg.NUM_BATCHES_TO_LOG_PROGRESS / elapsed
                    avg_throughput = throughput if avg_throughput is None else 0.5 * throughput + 0.5 * avg_throughput
                    eta = (steps - done) * cfg.TRAIN_BATCH_SIZE / avg_throughput
                    self.log("Train: during epoch #{epoch} batch {batch}/{tot_batches} ({batch_precision}%) -- "
                             "throughput (#samples/sec): {throughput} -- epoch ETA: {epoch_ETA} -- loss: {loss:.4f}".format(
                                 epoch=epoch + 1, batch=done, batch_precision=int(done / steps * 100), tot_batches=steps,
                                 throughput=int(throughput), epoch_ETA=str(datetime.timedelta(seconds=int(eta))),
                                 loss=window_loss / cfg.NUM_BATCHES_TO_LOG_PROGRESS))
                    window_loss, window_start = 0.0, time.time()
                if cfg.is_testing and done % cfg.NUM_TRAIN_BATCHES_TO_EVALUATE == 0:
                    self._evaluate_and_log()
            self.nr_epochs_trained = epoch + 1
            self.log("Completed epoch #{}: {}".format(epoch + 1, {"loss": epoch_loss / max(steps, 1)}))
            if cfg.is_saving and self.nr_epochs_trained - last_saved_epoch >= cfg.SAVE_EVERY_EPOCHS:
                self.log("Saving model after {} epochs.".format(self.nr_epochs_trained))
                self.save()
                self.log("Done saving model.")
                last_saved_epoch = self.nr_epochs_trained
            if cfg.is_testing:
                self._evaluate_and_log()

    def _evaluate_and_log(self):
        """ModelEvaluationCallback.perform_evaluation (keras_model.py:347-371)."""
        if self._avg_eval_duration is None:
            self.log("Evaluating...")
        else:
            self.log("Evaluating... (takes ~{})".format(str(datetime.timedelta(seconds=int(self._avg_eval_duration)))))
        start = time.time()
        res = self.evaluate()
        took = time.time() - start
        self._avg_eval_duration = took if self._avg_eval_duration is None else 0.5 * took + 0.5 * self._avg_eval_duration
        self.log("Done evaluating (took {}). Evaluation results:".format(str(datetime.timedelta(seconds=int(took)))))
        self.log("    loss: {loss:.4f}, f1: {f1:.4f}, recall: {recall:.4f}, precision: {precision:.4f}".format(
            loss=res.loss, f1=res.subtoken_f1, recall=res.subtoken_recall, precision=res.subtoken_precision))
        formatted = ["top{}: {:.4f}".format(i, acc) for i, acc in enumerate(res.topk_acc, start=1)]
        for chunk in common.chunks(formatted, 5):
            self.log("    " + ", ".join(chunk))

    # ---- evaluate: keras_eval_model.evaluate with the metrics of keras_model.py:96-113 ------------------
    def evaluate(self) -> Optional[ModelEvaluationResults]:
        import torch
        cfg = self.config
        if self.eval_reader is None:
            self.eval_reader = PathContextReader(vocabs=self.vocabs, model_input_tensors_former=_KerasEvaluateInputFormer(),
                                                 config=cfg, estimator_action=EstimatorAction.Evaluate)
        e = self.engine
        e.set_option("math_mode", self._math_eval)
        k = cfg.TOP_K_WORDS_CONSIDERED_DURING_PREDICTION
        oov = self.vocabs.target_vocab.special_words.OOV
        hits = np.zeros(k, dtype=np.float64)
        counts = SubtokenCounts()
        n_examples, loss_sum = 0, 0.0
        for batch in _prefetch(self.eval_reader.get_dataset()):
            t = _KerasEvaluateInputFormer().from_model_input_form(batch)
            idx, _probs, code_vectors, _ = e.predict_batch_host(
                t.path_source_token_indices, t.path_indices, t.path_target_token_indices, t.context_valid_mask,
                normalize=2, want_code=True, want_attention=False)
            B = int(idx.shape[0])
            target = np.asarray(t.target_index, dtype=np.int32).reshape(B)
            # mean cross entropy of the batch; Keras averages batch means weighted by batch size
            batch_loss = float(e.loss(e.to_device(code_vectors, torch.float32), e.to_device(target, torch.int32)).cpu()[0])
            loss_sum += batch_loss * B
            n_examples += B
            match = idx == target[:, None]                      # sparse_top_k_categorical_accuracy, k = 1..K
            hits += np.cumsum(match, axis=1).clip(max=1).sum(axis=0)[:k]
            top_words = self.vocabs.target_vocab.lookup_word(idx)
            for true_word, words in zip(t.target_string, top_words):
                legal = [w for w in words if w != oov and _LEGAL_WORD.match(w)]
                if legal:                                       # first legal predicted word (:88-106)
                    counts.update(common.binary_to_string(true_word), legal[0])
        if n_examples == 0:
            return None
        return ModelEvaluationResults(topk_acc=list(hits / n_examples), subtoken_precision=counts.precision,
                                      subtoken_recall=counts.recall, subtoken_f1=counts.f1, loss=loss_sum / n_examples)

    _PREDICT_NORMALIZE = 2                     # the device predict route's scores: full-vocabulary probabilities

    # ---- predict (keras_model.py:196-232): scores are full-vocabulary probabilities ---------------------
    def predict(self, predict_data_lines: Iterable[str]) -> List[ModelPredictionResults]:
        if self.predict_reader is None:
            self.predict_reader = PathContextReader(vocabs=self.vocabs, model_input_tensors_former=_EvaluateInputFormer(),
                                                    config=self.config, estimator_action=EstimatorAction.Predict)
        results: List[ModelPredictionResults] = []
        self.engine.set_option("math_mode", self._math_eval)
        for line in predict_data_lines:
            t = _EvaluateInputFormer().from_model_input_form(self.predict_reader.process_input_row(line))
            idx, probs, code_vectors, attn = self.engine.predict_batch_host(
                t.path_source_token_indices, t.path_indices, t.path_target_token_indices, t.context_valid_mask,
                normalize=2, want_code=True, want_attention=True)
            attention_per_context = self._get_attention_weight_per_context(
                t.path_source_token_strings[0], t.path_strings[0], t.path_target_token_strings[0], attn[0])
            results.append(ModelPredictionResults(
                original_name=common.binary_to_string(t.target_string[0]),
                topk_predicted_words=self.vocabs.target_vocab.lookup_word(idx[0]), topk_predicted_words_scores=probs[0],
                attention_per_context=attention_per_context, code_vector=code_vectors[0]))   # always set (:230)
        return results
