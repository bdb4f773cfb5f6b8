"""granne_b200 — H100-native drop-in for granne's search path (Granne::search and the Index / ElementContainer
read API), as hand-written sm_90a CUDA kernels behind the C ABI in include/granne_b200.h.

This package is a thin ctypes mirror of the reference's Python module (py/src/lib.rs:149-344 `Granne`): same
constructor arguments, same method names and defaults.  All computation happens in libgranne_b200.so on the GPU;
if the library is missing or no sm_90 (H100) device is present the calls fail loudly — there is no CPU fallback.
"""
from .api import (ANGULAR, ANGULAR_INT, EMBEDDINGS, QUERY_ELEMENT, QUERY_RAW_F32, BuildConfig, CsrLists, Granne,  # noqa: F401
                  GranneBuilder, GranneError, MultiGranne, PeerGather, elements_from_raw, elements_from_raw_device,
                  apply_order, compute_distance, compute_distances, compute_embeddings, compute_embeddings_and_save_to_disk,
                  compute_embeddings_device, compute_keys_for_reordering, decode_layer, inspect_index, library_path,
                  load_library, merge_topk_device, order_by_keys, order_from_trails, reencode_index)

from .words import Embeddings, WordDict  # noqa: F401,E402

__all__ = ["Embeddings", "WordDict", "CsrLists", "Granne", "GranneBuilder", "MultiGranne", "BuildConfig", "elements_from_raw", "elements_from_raw_device", "GranneError", "ANGULAR", "ANGULAR_INT", "EMBEDDINGS", "QUERY_RAW_F32", "QUERY_ELEMENT",
           "load_library", "library_path", "merge_topk_device", "inspect_index", "decode_layer", "reencode_index",
           "apply_order", "compute_distance", "compute_distances", "compute_embeddings", "compute_embeddings_device",
           "compute_embeddings_and_save_to_disk", "order_by_keys", "order_from_trails", "compute_keys_for_reordering"]
