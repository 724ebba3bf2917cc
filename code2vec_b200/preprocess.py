"""Offline dataset preparation (SURVEY section 8f, row N4): raw extractor output -> the `.c2v` files
and `.dict.c2v` the reader and the vocabularies consume.  Same command line, file formats and
sampling decisions as the reference's `preprocess.py` (file:line cited per function) plus the
histogram step its `preprocess.sh:56-58` delegates to awk, so a dataset can be produced without a
shell pipeline.  TensorFlow-free; byte-for-byte against the real reference in
tests/test_preprocess.py (golden files made by tests/golden/make_golden_preprocess.py).

A raw line is `target ctx ctx ...` with `ctx = token,path,token`; an output line has exactly
MAX_CONTEXTS context fields, padded with empty ones (SURVEY A.5).
"""
from __future__ import annotations

import os
import pickle
import random
from argparse import ArgumentParser
from collections import Counter
from typing import Dict, Iterable, List, Optional, Tuple


# ---- histograms (preprocess.sh:56-58: cut / tr / awk over the raw training file) -----------------
def count_histograms(train_data_path: str) -> Tuple[Counter, Counter, Counter]:
    """(token counts, path counts, target counts) of a raw training file.  Tokens are counted on both
    ends of every context, as `cut -d',' -f1,3 | tr ',' '\\n'` does."""
    tokens, paths, targets = Counter(), Counter(), Counter()
    with open(train_data_path, "r") as f:
        for line in f:
            fields = line.rstrip("\n").split(" ")
            targets[fields[0]] += 1
            for ctx in fields[1:]:
                parts = ctx.split(",")
                if len(parts) >= 3:
                    tokens[parts[0]] += 1
                    paths[parts[1]] += 1
                    tokens[parts[2]] += 1
                else:                         # malformed / empty field: awk still counts what cut gives it
                    tokens[parts[0]] += 1
                    if len(parts) > 1:
                        paths[parts[1]] += 1
    return tokens, paths, targets


def write_histogram(counts: Dict[str, int], path: str):
    """`word count` per line -- the format load_histogram reads."""
    with open(path, "w") as f:
        for word, n in counts.items():
            f.write("%s %d\n" % (word, n))


def load_histogram(path: str, max_size: Optional[int] = None) -> Dict[str, int]:
    """word -> count of the words that make the vocabulary (reference common.py:20-58, as
    preprocess.py:112-121 calls it: start_from=1, return_counts=True).

    Lines that are not exactly `word count` are skipped and a repeated word keeps its first count.
    If more than `max_size` words remain, the threshold is one more than the count of the word at
    rank max_size (0-based, descending), so words tied with it are dropped too -- the vocabulary can
    end up smaller than max_size, exactly as upstream."""
    def read(min_count: int) -> Dict[str, int]:
        kept: Dict[str, int] = {}
        with open(path, "r") as f:
            for line in f:
                cols = line.rstrip().split(" ")
                if len(cols) != 2:
                    continue
                n = int(cols[1])
                if n >= min_count and cols[0] not in kept:
                    kept[cols[0]] = n
        return kept

    counts = read(0)
    if max_size is None or len(counts) <= max_size:
        return counts
    return read(sorted(counts.values(), reverse=True)[max_size] + 1)


# ---- context down-sampling (preprocess.py:44-58,78-85) --------------------------------------------
def downsample_contexts(contexts: List[str], token_vocab, path_vocab, max_contexts: int, rng=random) -> List[str]:
    """At most `max_contexts` contexts of one method.  Contexts whose three parts are all in
    vocabulary are preferred; if those alone exceed the limit they are sampled, otherwise they are all
    kept and topped up with a sample of the partly known ones; wholly unknown contexts are dropped.
    A method within the limit is returned untouched (unknown contexts included)."""
    if len(contexts) <= max_contexts:
        return contexts
    full, partial = [], []
    for ctx in contexts:
        parts = ctx.split(",")
        known = (parts[0] in token_vocab, parts[1] in path_vocab, parts[2] in token_vocab)
        if all(known):
            full.append(ctx)
        elif any(known):
            partial.append(ctx)
    if len(full) > max_contexts:
        return rng.sample(full, max_contexts)
    if len(full) + len(partial) > max_contexts:
        return full + rng.sample(partial, max_contexts - len(full))
    return full + partial


def process_file(file_path: str, data_file_role: str, dataset_name: str, word_to_count, path_to_count,
                 max_contexts: int, rng=random, log=print) -> int:
    """Writes `<dataset_name>.<role>.c2v` and returns the number of examples kept (preprocess.py:23-75)."""
    seen_contexts = kept_contexts = written = empty = longest = 0
    with open("%s.%s.c2v" % (dataset_name, data_file_role), "w") as out, open(file_path, "r") as src:
        for line in src:
            fields = line.rstrip("\n").split(" ")
            target, contexts = fields[0], fields[1:]
            longest = max(longest, len(contexts))
            seen_contexts += len(contexts)
            contexts = downsample_contexts(contexts, word_to_count, path_to_count, max_contexts, rng)
            if not contexts:
                empty += 1
                continue
            kept_contexts += len(contexts)
            out.write(target + " " + " ".join(contexts) + " " * (max_contexts - len(contexts)) + "\n")
            written += 1
    log_file_stats(file_path, seen_contexts, kept_contexts, written, empty, longest, log)
    return written


def log_file_stats(file_path: str, seen_contexts: int, kept_contexts: int, written: int, empty: int, longest: int,
                   log=print):
    """process_file's report (preprocess.py:68-74); ZeroDivisionError when no example was written, as upstream."""
    log("File: " + file_path)
    log("Average total contexts: " + str(float(seen_contexts) / written))
    log("Average final (after sampling) contexts: " + str(float(kept_contexts) / written))
    log("Total examples: " + str(written))
    log("Empty examples: " + str(empty))
    log("Max number of contexts per word: " + str(longest))


def save_dictionaries(dataset_name: str, word_to_count, path_to_count, target_to_count, num_training_examples: int,
                      log=print):
    """`<dataset_name>.dict.c2v`: four consecutive pickles (preprocess.py:12-20; read back by
    vocabularies.py:220-230 and model_base.py:86-96)."""
    path = "%s.dict.c2v" % dataset_name
    with open(path, "wb") as f:
        for obj in (word_to_count, path_to_count, target_to_count, num_training_examples):
            pickle.dump(obj, f)
    log("Dictionaries saved to: " + path)


def arguments_parser() -> ArgumentParser:
    """The reference's flags (preprocess.py:88-110); the three histogram files become optional --
    when absent they are counted from the training file (what preprocess.sh:56-58 does with awk)."""
    p = ArgumentParser()
    p.add_argument("-trd", "--train_data", dest="train_data_path", required=True, help="path to training data file")
    p.add_argument("-ted", "--test_data", dest="test_data_path", required=True, help="path to test data file")
    p.add_argument("-vd", "--val_data", dest="val_data_path", required=True, help="path to validation data file")
    p.add_argument("-mc", "--max_contexts", dest="max_contexts", default=200, help="number of max contexts to keep")
    p.add_argument("-wvs", "--word_vocab_size", dest="word_vocab_size", default=1301136)
    p.add_argument("-pvs", "--path_vocab_size", dest="path_vocab_size", default=911417)
    p.add_argument("-tvs", "--target_vocab_size", dest="target_vocab_size", default=261245)
    p.add_argument("-wh", "--word_histogram", dest="word_histogram", metavar="FILE", default=None)
    p.add_argument("-ph", "--path_histogram", dest="path_histogram", metavar="FILE", default=None)
    p.add_argument("-th", "--target_histogram", dest="target_histogram", metavar="FILE", default=None)
    p.add_argument("-o", "--output_name", dest="output_name", metavar="FILE", required=True,
                   help="output name - the base name for the created dataset")
    return p


def main(argv: Optional[Iterable[str]] = None, rng=random, log=print) -> int:
    """C2V_DEVICE_PREPROCESS=1 runs the same command line on the GPU (device_preprocess.main); the files, the log lines
    of process_file and the state `rng` is left in are the same."""
    from .device_preprocess import device_preprocess_flag
    if device_preprocess_flag(os.environ):
        from . import device_preprocess
        return device_preprocess.main(argv, rng, log)
    args = arguments_parser().parse_args(None if argv is None else list(argv))
    histos = {"word": args.word_histogram, "path": args.path_histogram, "target": args.target_histogram}
    if not all(histos.values()):
        counted = dict(zip(("word", "path", "target"), count_histograms(args.train_data_path)))
        for kind, given in histos.items():
            if not given:
                histos[kind] = "%s.histo.%s.c2v" % (args.output_name, {"word": "ori", "path": "path", "target": "tgt"}[kind])
                write_histogram(counted[kind], histos[kind])
    word_to_count = load_histogram(histos["word"], int(args.word_vocab_size))
    path_to_count = load_histogram(histos["path"], int(args.path_vocab_size))
    target_to_count = load_histogram(histos["target"], int(args.target_vocab_size))
    num_training_examples = 0
    # test, val, train -- in this order, so the sampler's stream is consumed as upstream consumes it
    for file_path, role in ((args.test_data_path, "test"), (args.val_data_path, "val"), (args.train_data_path, "train")):
        n = process_file(file_path, role, args.output_name, word_to_count, path_to_count, int(args.max_contexts), rng, log)
        if role == "train":
            num_training_examples = n
    save_dictionaries(args.output_name, word_to_count, path_to_count, target_to_count, num_training_examples, log)
    return num_training_examples


if __name__ == "__main__":
    main()
