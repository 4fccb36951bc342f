"""A search session over several Trinity segments == IndexSourcesCollection (index_source.h:191-238, index_source.cpp:3-30).

Sources are ordered newest generation first; segment i is scanned with the updated_documents of every NEWER segment as its
masked-documents registry (fused into the emission stage on the device, trn_set_masked_documents); BM25 statistics are the
collection's (Σ docsCnt, Σ document frequency over the sources — similarity.h:202-222).  Each segment's postings live in HBM in
their own engine context; a query batch runs once per segment, exactly like the per-source exec_query() loop of a Trinity
application."""
from __future__ import annotations

import hashlib
import os
from typing import Dict, List, Optional, Sequence

import numpy as np

from . import (EMPTY_TERM, NODE_TERM, DocFilter, DocSet, GpuIndexSource, MergedSegment, MergeSource, Segment, TermDictionary, bm25_idf, parse_query)


def generation_of(path: str) -> int:
    """a segment directory's name is its generation (segment_index_source.cpp:18-21)"""
    return int(os.path.basename(os.path.normpath(str(path))))


class SegmentCollection:
    def __init__(self, paths: Sequence[str], device: int = 0, max_docid: int | None = None):
        paths = sorted((str(p) for p in paths), key=generation_of, reverse=True)
        self.paths = paths
        self.device = device
        self.generations = [generation_of(p) for p in paths]
        if len(set(self.generations)) != len(paths):
            raise ValueError("no two sources may share a generation")
        self.segments: List[Segment] = [Segment(p) for p in paths]
        self.dicts = [TermDictionary(s.names) for s in self.segments]
        self.docs_cnt = sum(s.field_statistics["docsCnt"] for s in self.segments)
        self._df = {}
        for s in self.segments:
            for n, t in zip(s.names, s.terms):
                self._df[n] = self._df.get(n, 0) + int(t["documents"])
        self.sources: List[GpuIndexSource] = []
        self._docsets: Dict[bytes, List[DocSet]] = {}  # the sets exec_batch registered, by content: one per source
        newer = np.zeros(0, np.uint32)
        for s in self.segments:
            g = GpuIndexSource(device)
            # the directory does not record the largest docID: 0 = the block directory built at upload finds it
            g.upload(s.codec, s.index, s.terms, max_docid or 0)
            if newer.size:
                g.set_masked_documents(newer)
            self.sources.append(g)
            if s.masked_documents.size:
                newer = np.union1d(newer, s.masked_documents).astype(np.uint32)

    def merge(self, out_codec: int, disable_optimizations: bool = False, device: int | None = None, payloads: bool = False) -> MergedSegment:
        """== MergeCandidatesCollection::merge over the collection's segments as they were opened (newest first, each masked by the
        updated documents of the newer ones) into one segment of out_codec; MergedSegment.write(path) persists it.  payloads=True:
        re-encoded hits keep their payloads (GpuIndexSource.merge_sources)"""
        srcs = [MergeSource.of_segment(s, p, g) for s, p, g in zip(self.segments, self.paths, self.generations)]
        g = GpuIndexSource(self.device if device is None else device)
        try:
            return g.merge_sources(out_codec, srcs, disable_optimizations, payloads)
        finally:
            g.close()

    def document_frequency(self, term: str) -> int:
        return self._df.get(term, 0)

    def plans(self, text: str, scored: bool):
        """one plan per segment (term ids are per dictionary); BM25 weights from the collection's statistics"""
        out = []
        for s, d in zip(self.segments, self.dicts):
            nodes = parse_query(text, d)
            if scored:
                for x in nodes:
                    if x["kind"] == NODE_TERM and x["term"] != EMPTY_TERM:
                        x["weight"] = bm25_idf(self._df[s.names[int(x["term"])]], self.docs_cnt)
            out.append(nodes)
        return out

    def intersect(self, token_groups: Sequence[Sequence[str]]):
        """== Trinity::intersect(0, tokens, collection) (intersect.cpp:172-201): every source's intersections with the updated documents of
        the newer sources masked, the tokens resolved per segment dictionary; concatenated, ordered by mask, equal masks summed"""
        acc = {}
        for g, d in zip(self.sources, self.dicts):
            for m, c in g.intersect_tokens(token_groups, d):
                acc[m] = acc.get(m, 0) + c
        return sorted(acc.items())

    def docsets(self, docids) -> List[DocSet]:
        """the docID set of these (global) docIDs in every source, collection order; a set passed again is the one registered before"""
        d = np.unique(np.asarray(docids, dtype=np.uint32))
        key = hashlib.sha1(d.tobytes()).digest()
        if key not in self._docsets:
            self._docsets[key] = [g.docset(d) for g in self.sources]
        return self._docsets[key]

    def release_docsets(self):
        """destroy every set exec_batch / docsets registered (each is a bitmap of the docID space in every source)"""
        for sets in self._docsets.values():
            for d in sets:
                d.close()
        self._docsets.clear()

    def filters(self, nq: int, allow=None, deny=None) -> Optional[List[List[Optional[DocFilter]]]]:
        """per source, one DocFilter (or None) per query from per-query allow / deny docID arrays (None: that side is open); None when no
        query has either"""
        allow = [None] * nq if allow is None else list(allow)
        deny = [None] * nq if deny is None else list(deny)
        if len(allow) != nq or len(deny) != nq:
            raise ValueError("allow / deny: one entry (or None) per query")
        if all(a is None for a in allow) and all(d is None for d in deny):
            return None
        per = [[None] * nq for _ in self.sources]
        for q in range(nq):
            a = self.docsets(allow[q]) if allow[q] is not None else None
            d = self.docsets(deny[q]) if deny[q] is not None else None
            if a is None and d is None:
                continue
            for i in range(len(self.sources)):
                per[i][q] = DocFilter(a[i] if a else None, d[i] if d else None)
        return per

    def exec_batch(self, queries: Sequence[str], mode: int, k: int = 100, allow=None, deny=None):
        """-> [BatchResult per segment], collection order (newest first).  allow / deny: per query None or an array of global docIDs
        (docIDs are global across generations: every source registers the same set, and a set passed again is reused)"""
        from . import MODE_DOCS_ONLY
        scored = mode != MODE_DOCS_ONLY
        per_q = [self.plans(q, scored) for q in queries]
        f = self.filters(len(queries), allow, deny)
        return [g.exec_batch([pq[i] for pq in per_q], mode, k, filters=None if f is None else f[i]) for i, g in enumerate(self.sources)]
