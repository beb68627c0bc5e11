"""
Tensor / logging / process-group helpers.

API parity with ``gossip/utils/helpers.py`` (flatten_tensors :21-36,
unflatten_tensors :39-57, group_by_dtype :60-70, communicate :73-88,
make_logger :91-114, is_power_of :117-128, create_process_group :131-146).
On the H100 hot path none of the flatten helpers run: parameters live in a
flat arena (``utils/arena.py``) and "flatten" is the identity.
"""

import collections
import logging
import sys

import torch
import torch.distributed as dist


def flatten_tensors(tensors):
    """One contiguous 1-D copy of same-dtype dense tensors.  If the tensors are
    already consecutive views of one storage (the arena case) the copy is a
    single memcpy of that span instead of a multi-source gather."""
    tensors = list(tensors)
    if len(tensors) == 1:
        return tensors[0].reshape(-1).clone()
    span = contiguous_span(tensors)
    if span is not None:
        return span.clone()
    return torch.cat([t.reshape(-1) for t in tensors], dim=0)


def contiguous_span(tensors):
    """If ``tensors`` are back-to-back contiguous views of one storage, return
    the 1-D view covering all of them (no copy); else None."""
    tensors = list(tensors)
    if not tensors:
        return None
    first = tensors[0]
    if not first.is_contiguous():
        return None
    try:
        base_ptr = first.untyped_storage().data_ptr()
    except Exception:
        return None
    offset = first.storage_offset()
    total = 0
    for t in tensors:
        if (t.dtype != first.dtype or not t.is_contiguous()
                or t.untyped_storage().data_ptr() != base_ptr
                or t.storage_offset() != offset + total):
            return None
        total += t.numel()
    return first.as_strided((total,), (1,), offset)


def unflatten_tensors(flat, tensors):
    """Views of ``flat`` shaped like ``tensors`` (no copies)."""
    outputs, offset = [], 0
    for t in tensors:
        n = t.numel()
        outputs.append(flat.narrow(0, offset, n).view_as(t))
        offset += n
    return tuple(outputs)


def group_by_dtype(tensors):
    by_dtype = collections.defaultdict(list)
    for t in tensors:
        by_dtype[t.dtype].append(t)
    return by_dtype


def communicate(tensors, communication_op):
    """flatten -> one collective per dtype -> scatter the result back."""
    for dtype, group in group_by_dtype(tensors).items():
        span = contiguous_span(group)
        if span is not None:           # arena-resident: communicate in place
            communication_op(tensor=span)
            continue
        flat = flatten_tensors(group)
        communication_op(tensor=flat)
        for f, t in zip(unflatten_tensors(flat, group), group):
            t.copy_(f)


_LOG_FORMAT = ': %(levelname)s -- %(threadName)s -- %(message)s'


def make_logger(rank, verbose=True, name=None):
    """Per-process stdout logger ``"{rank}: LEVEL -- thread -- msg"``;
    ``verbose`` -> DEBUG else INFO (set once, like the reference)."""
    logger = logging.getLogger(name or __name__)
    if not getattr(logger, 'handler_set', None):
        console = logging.StreamHandler(stream=sys.stdout)
        console.setFormatter(logging.Formatter(str(rank) + _LOG_FORMAT))
        logger.addHandler(console)
        logger.propagate = False
        logger.handler_set = True
    if not getattr(logger, 'level_set', None):
        logger.setLevel(logging.DEBUG if verbose else logging.INFO)
        logger.level_set = True
    return logger


def is_power_of(N, k):
    """True iff N == k**j for some integer j >= 0 (exact integer arithmetic)."""
    assert isinstance(N, int) and isinstance(k, int)
    assert k >= 0 and N > 0
    if N == 1:
        return True
    if k in (0, 1):
        return False
    while N % k == 0:
        N //= k
    return N == 1


def create_process_group(ranks):
    """``dist.new_group`` + a 1-element all-reduce so the (lazy) communicator
    exists before it is needed on the critical path."""
    group = dist.new_group(ranks)
    if dist.get_rank() in ranks:
        backend = dist.get_backend(group)
        dev = 'cuda' if (backend == 'nccl' and torch.cuda.is_available()) else 'cpu'
        dist.all_reduce(torch.ones(1, device=dev), group=group)
    return group
