"""How the golden files keep a recorded tensor, and how a run is compared with it.

A tensor is kept as the SHA-256 of its bytes (`<key>.sha256`: bit equality) and, for comparisons within a tolerance,
either whole (`<key>`: up to SMALL elements, or where the file names it so) or as a sketch (`<key>.sketch`): its rows
times a fixed Gaussian matrix of SKETCH_COLS columns, computed in float64 and stored as fp32.  A random projection keeps
the norm of a difference to within a small factor, so the relative error of the sketches stands for the relative error of
the tensors, and a [256, 128] gradient takes 16 KiB instead of 128 KiB of incompressible bytes.

Two digests are in the committed files, over different bytes, and neither may change:
- `sha256_tagged`: the dtype string, then the array's bytes in its own dtype (the `<key>.sha256` fields);
- `sha256_fp32`: the array's bytes as fp32, untagged (initial states `init_sha256.*` and the random draws)."""
import hashlib

import numpy as np

SMALL = 4096
SKETCH_COLS = 16


def sha256_tagged(a) -> str:
    """SHA-256 of the dtype string and the array's bytes in its own dtype (float64 stays float64)."""
    a = np.ascontiguousarray(a)
    return hashlib.sha256(a.dtype.str.encode() + a.tobytes()).hexdigest()


def sha256_fp32(a) -> str:
    """SHA-256 of the array's bytes as fp32, without a dtype tag."""
    return hashlib.sha256(np.ascontiguousarray(a, dtype=np.float32).tobytes()).hexdigest()


def sketch(a) -> np.ndarray:
    a = np.asarray(a, dtype=np.float64)
    a = a.reshape(a.shape[0], -1)
    R = np.random.default_rng(a.shape[1]).standard_normal((a.shape[1], SKETCH_COLS))
    return (a @ R).astype(np.float32)


def put_sha(g: dict, key: str, a):
    g[key + ".sha256"] = np.array(sha256_tagged(a))


def put(g: dict, key: str, a, whole: bool = False):
    """Record `a` under `key`: its digest, and the tensor itself or its sketch."""
    a = np.asarray(a)
    put_sha(g, key, a)
    if whole or a.size <= SMALL:
        g[key] = a.copy()
    else:
        g[key + ".sketch"] = sketch(a)


def equal(gold, key, a) -> bool:
    """`a` has the recorded bits (dtype and shape included)."""
    return sha256_tagged(np.asarray(a)) == str(gold[key + ".sha256"])


def rel(gold, key, a) -> float:
    """Relative 2-norm difference of `a` from the recorded tensor, or of their sketches."""
    a = np.asarray(a, dtype=np.float64)
    if key in gold:
        ref, got = np.asarray(gold[key], dtype=np.float64), a
    else:
        ref, got = np.asarray(gold[key + ".sketch"], dtype=np.float64), sketch(a)
    return float(np.linalg.norm(got - ref) / max(np.linalg.norm(ref), 1e-30))


def rel_to(a, ref) -> float:
    """Relative 2-norm difference of `a` from the array `ref`, the norm of `ref` taken in `ref`'s own dtype: how the files
    that keep their tensors whole (SLMRec, SELFCFED_LGN, MVGAE, LGMRec, MMGCN) have always been compared."""
    return float(np.linalg.norm(np.asarray(a, dtype=np.float64) - ref) / max(np.linalg.norm(ref), 1e-30))


def recorded(gold, prefix: str) -> list:
    """The keys recorded under `prefix` (e.g. "grad."), without the `.sha256` / `.sketch` suffixes."""
    keys = {str(k) for k in (gold.files if hasattr(gold, "files") else gold)}
    return sorted({k[:-len(".sha256")] for k in keys if k.startswith(prefix) and k.endswith(".sha256")})


def init_digests(model, plain=None) -> dict:
    """`sha256_fp32` of every `state_dict` entry (`param0.<name>`), then of each tensor in `plain` (`plain.<name>`): the
    tensors a model keeps beside its parameters.  Equal digests are equal bits."""
    out = {"param0." + k: sha256_fp32(v.detach().cpu().numpy()) for k, v in model.state_dict().items()}
    out.update({"plain." + k: sha256_fp32(v.detach().cpu().numpy()) for k, v in (plain or {}).items()})
    return out


def same_init(model, gold, plain=None) -> list:
    """Names of the initial states whose digest differs from the recorded one (empty: bit-identical), or whose set differs."""
    keys = gold.files if hasattr(gold, "files") else gold
    want = {str(k)[len("init_sha256."):]: str(gold[k]) for k in keys if str(k).startswith("init_sha256.")}
    got = init_digests(model, plain)
    return sorted(k for k in set(want) | set(got) if want.get(k) != got.get(k))
