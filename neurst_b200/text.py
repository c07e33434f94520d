"""Line-aligned parallel text files: the reader of the `ParallelTextDataset` class (neurst/data/datasets/
parallel_text_dataset.py:36-158).  Each line has its whitespace collapsed to single spaces; the target file is read
line by line beside the source file."""
import os


class ParallelTextDataset:
    """dataset.params: src_file, trg_file (optional for inference), data_is_processed.  `status` is the reference's
    data status: "processed" (BPE'd text, the recipes' `data_is_processed: True`) or "raw"."""

    def __init__(self, args):
        self.src_file = args.get("src_file")
        self.trg_file = args.get("trg_file")
        if not self.src_file:
            raise ValueError("ParallelTextDataset needs dataset.params.src_file")
        for p in (self.src_file, self.trg_file):
            if p and not os.path.isfile(p):
                raise FileNotFoundError("ParallelTextDataset: no such file %r" % p)
        self.processed = bool(args.get("data_is_processed", False))
        self._num_samples = None

    @property
    def status(self):
        s = "processed" if self.processed else "raw"
        return {"feature": s, "label": s}

    @property
    def num_samples(self):
        if self._num_samples is None:
            with open(self.src_file, encoding="utf-8") as f:
                self._num_samples = sum(1 for _ in f)
        return self._num_samples

    def build_iterator(self, map_func=None, shard_id=0, total_shards=1):
        """-> generator function over {"feature": text[, "label": text]} (build_iterator, :116-158), including its
        sharding rule: shard k keeps the 1-based line numbers n with begin_k <= n < end_k, where begin_k = k * (N //
        shards), end_k = begin_{k+1} and the last shard runs to the end."""
        if total_shards > 1:
            per = self.num_samples // total_shards
            begin = per * shard_id
            end = self.num_samples + 1 if shard_id == total_shards - 1 else begin + per

        def gen():
            with open(self.src_file, encoding="utf-8") as fsrc:
                ftrg = open(self.trg_file, encoding="utf-8") if self.trg_file else None
                try:
                    n = 0
                    for src in fsrc:
                        n += 1
                        data = {"feature": " ".join(src.strip().split())}
                        if ftrg is not None:
                            data["label"] = " ".join(ftrg.readline().strip().split())
                        if total_shards > 1:
                            if n < begin:
                                continue
                            if n >= end:
                                break
                        yield map_func(data) if map_func is not None else data
                finally:
                    if ftrg is not None:
                        ftrg.close()
        return gen
