"""Host-side pieces of `Code2VecModel` on 2, 4 or 8 GPUs (`python -m torch.distributed.run --nproc-per-node W -m
code2vec_b200 ...`, the fully sharded schedule): which runs are refused, how each rank takes its slice of a global batch,
and the `.c2v_b200` checkpoint written and read by several ranks at once.  Nothing here touches a GPU (DESIGN.md §6c).

Checkpoint layout (one format for every world size): magic, the header length (<Q), the json header, then the float32
tensors theta/*, adam_m/*, adam_v/* of the WHOLE model in PARAM_NAMES order.  A rank of a fully sharded run holds
  tok, path : the rows r with r % world == rank, as local rows r // world of a shard of ceil(T / world) rows (the tail
              of the shard past the table's end is padding and is never written or read);
  tgt       : the contiguous block [target_row0, target_row0 + rows) (trainer.target_row_block);
  W, a      : replicated; rank 0 writes them.
so each rank writes and reads only its own rows, and a file written on W ranks is the one a single GPU writes."""
from __future__ import annotations

import json
import os
import struct
from typing import Dict, List, Tuple

import numpy as np

from .engine import PARAM_NAMES, EngineDims

WORLD_SIZES = (1, 2, 4, 8)
CKPT_MAGIC = b"C2VB200\0"
CKPT_SUFFIX = ".c2v_b200"
_TF_NAMES = {"tok": "model/WORDS_VOCAB", "path": "model/PATHS_VOCAB", "tgt": "model/TARGET_WORDS_VOCAB",
             "W": "model/TRANSFORM", "a": "model/ATTENTION"}


# ---- launch ------------------------------------------------------------------------------------------------------------
def run_world(environ) -> Tuple[int, int]:
    """(world size, local rank) of this process as torch.distributed.run sets them; (1, 0) outside a launcher."""
    return int(environ.get("WORLD_SIZE", "1") or "1"), int(environ.get("LOCAL_RANK", "0") or "0")


def check_multi_rank_run(config, world: int, save_format: str = "c2v_b200") -> None:
    """Raises ValueError if `config` (saving in `save_format`, tf_bundle.save_format_flag) cannot run on `world` ranks.
    Host only: it runs before any engine exists."""
    if world not in WORLD_SIZES:
        raise ValueError("WORLD_SIZE=%d: Code2VecModel runs on 1, 2, 4 or 8 GPUs (the embedding tables are row-sharded "
                         "over the ranks); launch with --nproc-per-node 2, 4 or 8" % world)
    if world == 1:
        return
    if config.TRAIN_BATCH_SIZE % world:
        raise ValueError("TRAIN_BATCH_SIZE=%d is not a multiple of the %d ranks: every rank takes an equal slice of each "
                         "global batch; choose a batch size divisible by %d" % (config.TRAIN_BATCH_SIZE, world, world))
    if config.PREDICT:
        raise ValueError("--predict runs on one GPU: load the saved model in a single process (without "
                         "torch.distributed.run), which reads a checkpoint saved on any number of GPUs")
    if config.RELEASE:
        raise ValueError("--release runs on one GPU: load the saved model in a single process (without "
                         "torch.distributed.run), which reads a checkpoint saved on any number of GPUs")
    if config.DL_FRAMEWORK == "b200-keras":
        raise ValueError("--framework b200-keras runs on one GPU: train on several GPUs with --framework b200, or run "
                         "the Keras backend in a single process")
    if save_format != "c2v_b200":
        raise ValueError("C2V_SAVE_FORMAT=%s: TensorFlow checkpoints are written by one GPU; save .c2v_b200 checkpoints "
                         "on several GPUs (unset C2V_SAVE_FORMAT), then load and save (or --release) in a single process "
                         "with C2V_SAVE_FORMAT=%s" % (save_format, save_format))


def batch_split(rows: int, world: int, rank: int) -> Tuple[int, int, int]:
    """(lo, hi, dropped): rank `rank` takes rows [lo, hi) of a global batch of `rows` rows.  Every rank takes
    floor(rows / world) rows, so a short batch runs as a step of world * floor(rows / world) rows and its last `dropped`
    (< world) rows are left out; with rows < world no rank takes any."""
    b = rows // world
    return rank * b, (rank + 1) * b, rows - world * b


# ---- checkpoint --------------------------------------------------------------------------------------------------------
def checkpoint_header(dims: dict, adam_t: int, epochs_trained: int, with_optimizer: bool):
    """(file prefix = magic + length + json header, [tensor entries], total file size) of a checkpoint of a model with
    the GLOBAL dims `dims` (vars(EngineDims)).  Entries: {"name", "shape", "offset", "nbytes"}, offsets from the end of
    the prefix."""
    shapes = EngineDims(**dims).shapes()
    groups = ("theta", "adam_m", "adam_v") if with_optimizer else ("theta",)
    meta = {"format": 1, "dims": dict(dims), "adam_t": int(adam_t) if with_optimizer else 0,
            "epochs_trained": int(epochs_trained), "tf_names": dict(_TF_NAMES), "tensors": []}
    offset = 0
    for g in groups:
        for k in PARAM_NAMES:
            n = int(np.prod(shapes[k])) * 4
            meta["tensors"].append({"name": g + "/" + k, "shape": list(shapes[k]), "offset": offset, "nbytes": n})
            offset += n
    header = json.dumps(meta).encode()
    prefix = CKPT_MAGIC + struct.pack("<Q", len(header)) + header
    return prefix, meta["tensors"], len(prefix) + offset


def write_checkpoint(path: str, prefix: bytes, arrays: List[np.ndarray]) -> None:
    """One process holding every tensor: the prefix, then the arrays (in the header's order) as little-endian float32."""
    with open(path, "wb") as f:
        f.write(prefix)
        for a in arrays:
            f.write(np.asarray(a).astype("<f4", copy=False).tobytes())


def create_checkpoint_file(path: str, prefix: bytes, total: int) -> None:
    """Rank 0 of a sharded save: the prefix, and the file sized for every tensor (the ranks fill the rows in)."""
    with open(path, "wb") as f:
        f.write(prefix)
        f.truncate(total)


def _tensor_map(path: str, base: int, ent: dict, mode: str):
    return np.memmap(path, dtype="<f4", mode=mode, offset=base + ent["offset"], shape=tuple(ent["shape"]))


def _own_rows(name: str, m, rank: int, world: int, target_rows: Tuple[int, int]):
    """The part of the whole tensor `m` this rank holds (see the module docstring)."""
    if name in ("tok", "path"):
        return m[rank::world]
    if name == "tgt":
        return m[target_rows[0]:target_rows[1]]
    return m


def write_checkpoint_part(path: str, prefix_len: int, entries: List[dict], rank: int, world: int,
                          target_rows: Tuple[int, int], local: Dict[str, np.ndarray]) -> None:
    """This rank's rows of the tensors in `local` ({"theta/tok": shard, "theta/tgt": block, ...}) into a file made by
    create_checkpoint_file.  Shards may carry padding rows past the table's end; they are not written.  W and a only
    from rank 0."""
    for ent in entries:
        name = ent["name"].split("/")[1]
        if ent["name"] not in local or (name in ("W", "a") and rank != 0):
            continue
        m = _tensor_map(path, prefix_len, ent, "r+")
        dst = _own_rows(name, m, rank, world, target_rows)
        src = np.asarray(local[ent["name"]], dtype=np.float32)
        if dst.ndim:
            src = src[:dst.shape[0]]
        dst[...] = src.reshape(dst.shape)
        m.flush()
        del m


def read_checkpoint_header(path: str):
    """(header dict, prefix length) of a checkpoint file; ValueError if it is missing or not one."""
    if not os.path.isfile(path):
        raise ValueError("There is no model at path `{}`.".format(path))
    with open(path, "rb") as f:
        if f.read(8) != CKPT_MAGIC:
            raise ValueError("`{}` is not a c2v_b200 checkpoint".format(path))
        (hlen,) = struct.unpack("<Q", f.read(8))
        return json.loads(f.read(hlen).decode()), 16 + hlen


def read_checkpoint_part(path: str, rank: int, world: int, target_rows: Tuple[int, int], out: dict) -> dict:
    """This rank's rows of every tensor named in `out` into out[name] (numpy array or torch tensor, shard-shaped: its
    first rows are filled, padding rows are left as they are).  Tensors the file does not hold are left untouched.
    Returns the header."""
    meta, base = read_checkpoint_header(path)
    read_entries_part(path, base, meta["tensors"], rank, world, target_rows, out)
    return meta


def read_entries_part(path: str, base: int, entries: List[dict], rank: int, world: int, target_rows: Tuple[int, int],
                      out: dict) -> None:
    """read_checkpoint_part for tensor entries whose bytes start at `base` of `path` (or of ent["file"], when an entry
    names its own file)."""
    for ent in entries:
        dest = out.get(ent["name"])
        if dest is None:
            continue
        src = np.array(_own_rows(ent["name"].split("/")[1], _tensor_map(ent.get("file", path), base, ent, "r"), rank,
                                 world, target_rows))
        if isinstance(dest, np.ndarray):
            dest[:src.shape[0]] = src
        else:
            import torch
            dest[:src.shape[0]].copy_(torch.from_numpy(src))


def check_checkpoint_dims(meta: dict, dims: dict) -> None:
    """ValueError if the checkpoint's table sizes are not the model's."""
    for key in ("token_vocab", "path_vocab", "target_vocab", "embed_dim", "code_dim"):
        if meta["dims"][key] != dims[key]:
            raise ValueError("checkpoint %s=%s does not match the model (%s)" % (key, meta["dims"][key], dims[key]))
