"""Inputs of the typed VF-vGPU CDI spec tests (kxpu_cdi_emit_vf_vgpu[_cdev] / kxpu_cdi_parse_vf_vgpu[_cdev]): records with
a vGPU type ID and type key per device, over cdi_parse_cases' bdfs (base-60 quoted and plain), groups and indices."""
import numpy as np

import cdi_parse_cases as CP
from kxpu_b200.binding import CDEV_FIELD, VFVGPUCDI_DTYPE

FMT_YAML, FMT_JSON = CP.FMT_YAML, CP.FMT_JSON
KIND_3 = b"a/b"
KIND_14 = b"nvidia.com/gpu"
KIND_63 = CP.KIND_LONG
KINDS = [KIND_3, KIND_14, KIND_63]
# keys that a YAML 1.1 or 1.2 resolver (or JSON, unquoted) would read as something other than a string
TRICKY_KEYS = [b"true", b"No", b"1_000", b"0x1F", b".inf", b"1e5", b"2024-01-01", b"null", b"0o17", b"-.5", b"y", b"1"]
EDGE_KEYS = [b"A", b"k" * 40, b"NVIDIA_H100-4C", b"a.b-c_d"] + TRICKY_KEYS
EDGE_IDS = [1, (1 << 32) - 1, 557, 10, 9]


def records(n, seed=0):
    """n records: the edge IDs and keys first, then IDs over the whole range and keys of 1..40 bytes of the alphabet;
    cdev numbers of every width."""
    base = CP.records(n, False, seed)
    rng = np.random.default_rng(seed + 2000)
    a = np.zeros(n, VFVGPUCDI_DTYPE)
    a["dev"] = base
    a["dev"][CDEV_FIELD] = rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32)
    a["type_id"] = rng.integers(1, 1 << 32, n, dtype=np.uint64).astype(np.uint32)
    alphabet = np.frombuffer(b"ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789_.-", np.uint8)
    lens = rng.integers(1, 41, n)
    keys = np.zeros((n, 40), np.uint8)
    for i in range(min(n, 4096)):  # beyond that, one pattern per length keeps large cases quick
        keys[i, :lens[i]] = alphabet[rng.integers(0, len(alphabet), lens[i])]
    if n > 4096:
        pat = np.stack([np.pad(alphabet[np.arange(L) % len(alphabet)], (0, 40 - L)) for L in range(1, 41)])
        keys[4096:] = pat[lens[4096:] - 1]
    k = min(n, len(EDGE_KEYS))
    for i in range(k):
        keys[i] = 0
        keys[i, :len(EDGE_KEYS[i])] = np.frombuffer(EDGE_KEYS[i], np.uint8)
        lens[i] = len(EDGE_KEYS[i])
    a["key"] = keys.view("S40").reshape(n)
    a["key_len"] = lens
    a["type_id"][:min(n, len(EDGE_IDS))] = EDGE_IDS[:min(n, len(EDGE_IDS))]
    return a


def group_view(recs):
    """the records as the group layout's parser returns them: no cdev number"""
    out = recs.copy()
    out["dev"][CDEV_FIELD] = 0
    return out
