"""loro_b200 -- H100-native batched CRDT merge engine (one hot path of loro-dev/loro).

Host-side mirror of the reference's public API for that path (crates/loro/src/lib.rs):
  LoroDoc::import / import_batch  ->  import_batch(blobs)            (one fresh document per blob)
  ImportStatus                    ->  Batch.status(i)
  LoroDoc::get_deep_value         ->  Batch.get_deep_value(i)
  LoroDoc::oplog_vv / oplog_frontiers ->  Batch.oplog_vv(i) / Batch.oplog_frontiers(i)
  LoroDoc::export(ExportMode)     ->  Batch.export_updates(i, from_vv=None)   (all_updates / updates(from))
  import / import_batch on a document that already holds history  ->  DocSet.import_(blobs, doc_ids)
  LoroDoc::checkout(&frontiers) + get_deep_value  ->  import_batch_at(blobs, versions) / DocSet.checkout(requests)
All compute runs in the CUDA library built from loro_b200/csrc (C ABI: include/loro_b200.h).  There is no
CPU fallback: importing a batch without the built library or without a CUDA device raises.
"""
from .api import (Batch, MultiBatch, DocError, DocSet, EngineUnavailable, ImportStatus, import_batch, import_batch_at,
                  import_batch_device, library_path, load_library, numa_bind, device_trim, pack_blobs)

__all__ = ["Batch", "MultiBatch", "DocError", "DocSet", "EngineUnavailable", "ImportStatus", "import_batch", "import_batch_at",
           "import_batch_device", "library_path", "load_library", "numa_bind", "device_trim", "pack_blobs"]
