"""`python -m code2vec_b200 ...`: the reference's command line (code2vec.py:16-38) on the engine's backends.

Same flags (`Config.arguments_parser`, reference config.py:11-44) and the same order of actions:
train, export word2vec files, evaluate (or release), predict.  `--predict` differs in one respect: the
reference's REPL shells out to the Java path extractor (interactive_predict.py:18-21, extractor.py),
which is out of scope here; this entry point reads ALREADY-EXTRACTED lines (`name ctx ctx ...`, the
extractor's output format, SURVEY A.5) from `--predict_input FILE` or standard input, post-processes
them as extractor.py:22-38 does (first MAX_CONTEXTS contexts, path strings replaced by their Java
`String.hashCode`, padding to MAX_CONTEXTS fields) and prints each prediction in the reference's layout
(interactive_predict.py:50-63), attention paths un-hashed when the input carried path strings.
"""
from __future__ import annotations

import os
import sys
from typing import Iterable, Optional

import numpy as np

from . import load_model_dynamically, name_scores, similarity
from .common import common
from .config import Config
from .multi_rank import run_world
from .vocabularies import VocabType

SHOW_TOP_CONTEXTS = 10       # interactive_predict.py:6


def java_string_hashcode(s: str) -> int:
    """Java's String.hashCode (s[0]*31^(n-1) + ... + s[n-1] in wrapping 32-bit arithmetic) as a signed int:
    datasets store paths under this hash (extractor.py:40-49, ProgramRelation.java:18)."""
    h = 0
    for ch in s:
        h = (h * 31 + ord(ch)) % (1 << 32)
    return h - (1 << 32) if h >= (1 << 31) else h


def _looks_hashed(path: str) -> bool:
    body = path[1:] if path[:1] == "-" else path
    return body.isdigit()


def prepare_extracted_lines(lines: Iterable[str], max_contexts: int):
    """Extractor output -> model input lines + {hashed path: path string} (extractor.py:20-38)."""
    out, unhash = [], {}
    for line in lines:
        fields = line.rstrip().split(" ")
        if not fields or not fields[0]:
            continue
        contexts = [c for c in fields[1:] if c]
        kept = []
        for ctx in contexts[:max_contexts]:
            token1, path, token2 = ctx.split(",")
            hashed = path if _looks_hashed(path) else str(java_string_hashcode(path))
            unhash[hashed] = path
            kept.append("%s,%s,%s" % (token1, hashed, token2))
        out.append(" ".join([fields[0]] + kept) + " " * (max_contexts - len(kept)))
    return out, unhash


def print_predictions(config: Config, model, lines: Iterable[str], out=None):
    out = sys.stdout if out is None else out
    lines, unhash = prepare_extracted_lines(lines, config.MAX_CONTEXTS)
    if not lines:
        return
    raw_results = model.predict(lines)
    parsed = common.parse_prediction_results(raw_results, unhash, model.vocabs.target_vocab.special_words,
                                             topk=SHOW_TOP_CONTEXTS)
    for raw, method in zip(raw_results, parsed):
        out.write("Original name:\t" + method.original_name + "\n")
        for pair in method.predictions:
            out.write("\t(%f) predicted: %s\n" % (pair["probability"], pair["name"]))
        out.write("Attention:\n")
        for att in method.attention_paths:
            out.write("%f\tcontext: %s,%s,%s\n" % (att["score"], att["token1"], att["path"], att["token2"]))
        if config.EXPORT_CODE_VECTORS:
            out.write("Code vector:\n")
            out.write(" ".join(map(str, raw.code_vector)) + "\n")


def print_most_similar(model, vocab_type: VocabType, lines: Iterable[str], topn: int, out=None):
    """One block per query line (`pos1,pos2[ neg1,neg2]`): `Most similar to:\\t<line>`, then `\\t(%f) <word>` per result;
    a query with a word outside the vocabulary prints `Not in vocabulary: <w>` instead."""
    out = sys.stdout if out is None else out
    for line in lines:
        query = similarity.parse_query_line(line)
        if query is None:
            continue
        missing = [w for w in query[0] + query[1] if w not in model.vocabs.get(vocab_type).word_to_index]
        if missing:
            out.write("Not in vocabulary: %s\n" % missing[0])
            continue
        out.write(similarity.format_most_similar(line, model.most_similar(query[0], query[1], topn=topn,
                                                                          vocab_type=vocab_type)))


def write_nearest(model, c2v_path: str, topn: int) -> str:
    """`<c2v_path>.nearest`: line r is example r's name, then `\\t<row>,<name>,<similarity>` per nearest other example.
    With C2V_DEVICE_EVAL=1 the corpus is read, searched and the file written on the GPU (DESIGN.md §6o)."""
    if getattr(model, "device_eval", False):
        return model.write_nearest_device(c2v_path, topn)
    names, _vectors, idx, val = model.nearest_code_vectors(c2v_path, topn)
    out_path = c2v_path + ".nearest"
    pad = np.iinfo(np.int32).max
    with open(out_path, "w") as f:
        for r, name in enumerate(names):
            f.write(similarity.format_nearest_line(
                name, [(int(j), names[j], float(v)) for j, v in zip(idx[r], val[r]) if j != pad]))
    return out_path


def write_name_scores(model, c2v_path: str) -> str:
    """`<c2v_path>.name_scores`: one line per example evaluate() scores, in its order (name_scores.format_line); the
    summary line is logged.  With C2V_DEVICE_EVAL=1 the corpus is read, scored and the file written on the GPU (§6o)."""
    if getattr(model, "device_eval", False):
        return model.write_name_scores_device(c2v_path)
    names, target_ids, rank, logp, top1, top1_logp = model.score_names(c2v_path)
    vocab = model.vocabs.target_vocab
    in_vocab = target_ids != vocab.word_to_index[vocab.special_words.OOV]
    top1_names = vocab.lookup_word(top1)
    out_path = c2v_path + name_scores.SUFFIX
    with open(out_path, "w") as f:
        for r, name in enumerate(names):
            f.write(name_scores.format_line(name, bool(in_vocab[r]), int(rank[r]), float(logp[r]), top1_names[r],
                                            float(top1_logp[r])))
    model.config.log(name_scores.summary_line(rank, logp, in_vocab))
    return out_path


def main(argv: Optional[Iterable[str]] = None) -> int:
    argv = list(sys.argv[1:] if argv is None else argv)
    predict_input = None
    if "--predict_input" in argv:                      # the one flag the reference does not have
        i = argv.index("--predict_input")
        predict_input = argv[i + 1]
        del argv[i:i + 2]
    argv, sim = similarity.split_cli_flags(argv)       # --most_similar, --most_similar_input, --nearest, --topn
    argv, score_path = name_scores.split_cli_flags(argv)
    similarity.check_single_gpu(sim, run_world(os.environ)[0])
    name_scores.check_single_gpu(score_path, run_world(os.environ)[0])
    config = Config(set_defaults=True)
    config.load_from_args(argv)
    config.verify()
    model = load_model_dynamically(config)
    config.log("Done creating code2vec model")
    try:
        if config.is_training:
            model.train()
        if config.SAVE_W2V is not None:
            model.save_word2vec_format(config.SAVE_W2V, VocabType.Token)
            config.log("Origin word vectors saved in word2vec text format in: %s" % config.SAVE_W2V)
        if config.SAVE_T2V is not None:
            model.save_word2vec_format(config.SAVE_T2V, VocabType.Target)
            config.log("Target word vectors saved in word2vec text format in: %s" % config.SAVE_T2V)
        if (config.is_testing and not config.is_training) or config.RELEASE:
            eval_results = model.evaluate()
            if eval_results is not None:
                config.log(str(eval_results).replace("topk", "top{}".format(config.TOP_K_WORDS_CONSIDERED_DURING_PREDICTION)))
        if config.PREDICT:
            model.predict([])                          # the reference's warm-up call (interactive_predict.py:16)
            if getattr(model, "device_predict", False):
                # C2V_DEVICE_PREDICT=1: the whole input as bytes, read with the source's newline rule on the GPU
                if predict_input:
                    with open(predict_input, "rb") as f:
                        data, universal = f.read(), True
                else:
                    data, universal = sys.stdin.buffer.read(), False
                sys.stdout.flush()
                if model.print_predictions_device(data, universal, sys.stdout.buffer):
                    sys.stdout.buffer.flush()
                else:
                    from .device_predict import split_source_lines
                    print_predictions(config, model, split_source_lines(data, universal))
            elif predict_input:
                with open(predict_input, "r") as f:
                    print_predictions(config, model, f)
            else:
                print_predictions(config, model, sys.stdin)
        if sim.most_similar is not None:
            vocab_type = {"target": VocabType.Target, "token": VocabType.Token, "path": VocabType.Path}[sim.most_similar]
            if sim.most_similar_input:
                with open(sim.most_similar_input, "r") as f:
                    print_most_similar(model, vocab_type, f, sim.topn)
            else:
                print_most_similar(model, vocab_type, sys.stdin, sim.topn)
        if sim.nearest is not None:
            config.log("Nearest code vectors written to: %s" % write_nearest(model, sim.nearest, sim.topn))
        if score_path is not None:
            config.log("Name scores written to: %s" % write_name_scores(model, score_path))
    finally:
        model.close_session()
    return 0


if __name__ == "__main__":
    sys.exit(main())
