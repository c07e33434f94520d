"""Prune-Tune (examples/prune_tune, Liang et al., AAAI 2021): the mask files of a pruned model and of its partial tuning.

The reference pickles one `tf.Variable` per trainable variable into `<model_dir>/mask.pkl` (partial_trainer.py:188-206),
which nothing can read without TensorFlow.  Here the same file name holds a NumPy .npz archive instead: one uint8 0/1 array
per parameter tensor, in the tensor's shape, keyed by its reference variable name exactly as checkpoints.save_npz keys the
weights (1 = the weight is kept by the pruning, i.e. frozen by the partial tuning; 0 = pruned, i.e. tuned).  The loader
resolves the archive's top-level scope as checkpoints.load_npz does, so one file format serves the speech, text and wait-k
models, and it refuses a real pickle, missing or extra names, wrong shapes and values other than 0/1.

On the device the masks are the pruning's bitmap (Runtime.derive_prune_mask): bit j of byte b is element 8b + j of the
parameter arena, 1 in the alignment padding.
"""
import os

import numpy as np

from neurst_b200 import checkpoints as CK

MASK_FILE = "mask.pkl"


class MaskFileError(ValueError):
    """A mask file this path cannot use."""


def _numel(shape):
    n = 1
    for s in shape:
        n *= int(s)
    return n


def save_masks(rt, path, bitmap):
    """Writes the bits of `bitmap` (device or host uint8 [numel / 8], derive_prune_mask's layout) for every parameter tensor of
    `rt` to `path` as a NumPy .npz archive, whatever the file name (the recipe's is mask.pkl).  The file is replaced
    atomically."""
    bits = np.unpackbits(np.asarray(bitmap.cpu() if hasattr(bitmap, "cpu") else bitmap, dtype=np.uint8), bitorder="little")
    names = CK.tf_variable_names(rt.table)
    arrays = {names[k]: bits[off:off + _numel(shape)].reshape(shape) for k, (off, shape) in rt.table.items()}
    tmp = path + ".tmp"
    with open(tmp, "wb") as f:               # a file object: np.savez would append .npz to a file name
        np.savez(f, **arrays)
    os.replace(tmp, path)
    return sorted(arrays)


def load_masks(rt, path):
    """{our parameter name: uint8 0/1 array in the tensor's shape} from a mask file that save_masks wrote (or any .npz
    archive of that form).  Raises MaskFileError, with what is wrong, for anything else."""
    if not os.path.isfile(path):
        raise MaskFileError("mask_pkl %s: no such file" % path)
    with open(path, "rb") as f:
        head = f.read(4)
    if not head.startswith(b"PK"):
        if head[:1] == b"\x80":
            raise MaskFileError("mask_pkl %s is a Python pickle: the reference's mask.pkl holds TensorFlow variables, which "
                                "cannot be read without TensorFlow; this path needs the .npz form (one uint8 0/1 array per "
                                "reference variable name), which prune_tune_train writes" % path)
        raise MaskFileError("mask_pkl %s is not a NumPy .npz archive of masks" % path)
    try:
        z = np.load(path, allow_pickle=False)
        files = list(z.files)
        scope = CK.archive_scope(files, rt.table)
        names = CK.tf_variable_names(rt.table, scope)
        want = set(names.values())
        missing = sorted(want - set(files))
        extra = sorted(set(files) - want)
        if missing:
            raise MaskFileError("mask_pkl %s misses the masks of %d variables of the model, e.g. %s" % (path, len(missing), missing[:3]))
        if extra:
            raise MaskFileError("mask_pkl %s holds masks of %d variables the model does not have, e.g. %s" % (path, len(extra), extra[:3]))
        out = {}
        for k, v in names.items():
            a = z[v]
            shape = tuple(rt.table[k][1])
            if tuple(a.shape) != shape:
                raise MaskFileError("mask_pkl %s: the mask of %s has shape %s, the variable %s" % (path, v, tuple(a.shape), shape))
            if a.dtype.kind not in "biuf" or not ((a == 0) | (a == 1)).all():
                raise MaskFileError("mask_pkl %s: the mask of %s holds values other than 0 and 1" % (path, v))
            out[k] = a.astype(np.uint8)
        return out
    except MaskFileError:
        raise
    except (ValueError, OSError) as e:                  # a damaged archive, or an object array (allow_pickle=False)
        raise MaskFileError("mask_pkl %s: %s" % (path, e))


def mask_bitmap(rt, masks):
    """The device bitmap of {our name: 0/1 array} over every parameter tensor (Runtime.derive_prune_mask)."""
    return rt.derive_prune_mask(list(rt.table), masks)
