"""Index a corpus with the H100 engine.  Same flags and output format as the reference's
`retrieval/index.py` (--ckpt_path, --corpus-path, --output-path, --batch-size; writes a pickled
`IndexedCorpus` with fp32 CPU embeddings, retrieval/index.py:33-40), so the result can be
handed to anything that calls `load_corpus(indexed_corpus_path)`.

    python -m reprover_b200.index_cli --ckpt_path <hf dir> --corpus-path corpus.jsonl --output-path index.pickle

Under `torchrun --nproc-per-node N` (one process per GPU) the corpus is re-indexed row-sharded — every rank
encodes its N-th of the premises, no communication — and rank 0 gathers the rows and writes the same
single-file index (the reference has no counterpart: it indexes on one device, retrieval/index.py:26-33).
"""
from __future__ import annotations

import argparse
import logging

import torch

from .retriever import B200PremiseRetriever

logger = logging.getLogger("reprover_b200.index")


def main(argv=None) -> None:
    parser = argparse.ArgumentParser(description="Index a premise corpus with the H100 retrieval engine.")
    parser.add_argument("--ckpt_path", type=str, required=True)
    parser.add_argument("--corpus-path", type=str, required=True)
    parser.add_argument("--output-path", type=str, required=True)
    parser.add_argument("--batch-size", type=int, default=64)
    parser.add_argument("--max-seq-len", type=int, default=2048)  # the reference hard-codes 2048 (index.py:33)
    parser.add_argument("--native-layout", action="store_true",
                        help="pickle this package's own classes instead of the reference's layout")
    args = parser.parse_args(argv)
    logging.basicConfig(level=logging.INFO)
    logger.info(args)
    if not torch.cuda.is_available():
        # the reference falls back to the CPU with a warning (index.py:28-30); this engine does not
        raise SystemExit("reprover_b200 needs an H100 GPU: there is no CPU indexing path")
    import os

    world = int(os.environ.get("WORLD_SIZE", "1"))
    if world > 1:
        import torch.distributed as dist

        local = int(os.environ.get("LOCAL_RANK", "0"))
        torch.cuda.set_device(local)
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
        model = B200PremiseRetriever.load_hf(args.ckpt_path, args.max_seq_len, torch.device("cuda", local))
        model.load_corpus(args.corpus_path)
        index = model.reindex_corpus_sharded(batch_size=args.batch_size)
        indexed = index.gather_indexed_corpus(model.corpus, dst=0)       # fp32 CPU rows on rank 0
        if dist.get_rank() == 0:
            model.corpus_embeddings = indexed.embeddings
            model.embeddings_staled = False
            model.save_index(args.output_path, reference_layout=not args.native_layout)
            logger.info("Indexed corpus (%d ranks) saved to %s", world, args.output_path)
        dist.barrier()
        dist.destroy_process_group()
        return
    model = B200PremiseRetriever.load_hf(args.ckpt_path, args.max_seq_len, torch.device("cuda"))
    model.load_corpus(args.corpus_path)
    model.reindex_corpus(batch_size=args.batch_size)
    model.save_index(args.output_path, reference_layout=not args.native_layout)
    logger.info("Indexed corpus saved to %s", args.output_path)


if __name__ == "__main__":
    main()
