"""sourmash_b200 -- H100-native FracMinHash sketching and sorted-hash intersection.

Drop-in for the two hot paths of sourmash (DESIGN.md, include/sourmash_b200.h):

    from sourmash_b200 import MinHash, SourmashSignature          # object model over the C ABI
    from sourmash_b200.compare import compare_all_pairs           # N x N on the GPU
    from sourmash_b200.index import LinearIndex, CounterGather    # search / prefetch / gather
    from sourmash_b200 import batch                               # raw batched entry points
"""
from . import batch  # noqa: F401
from ._lowlevel import ffi, lib  # noqa: F401
from .minhash import (FrozenMinHash, MinHash, get_minhash_default_seed, get_minhash_max_hash,  # noqa: F401
                      hash_murmur, translate_codon)
from .signature import (ComputeParameters, SourmashSignature, load_one_signature_from_json, load_signatures,  # noqa: F401
                        load_signatures_from_json, save_signatures_to_json)

# the names the reference's __init__ still exports for these (sourmash/__init__.py:47-100; deprecated there)
from .index import load_file_as_index, load_file_as_signatures  # noqa: E402,F401

load_one_signature = load_one_signature_from_json
save_signatures = save_signatures_to_json
DEFAULT_SEED = get_minhash_default_seed()
MAX_HASH = get_minhash_max_hash()

__version__ = "0.1.0"
