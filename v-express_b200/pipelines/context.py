"""Context-window scheduler: drop-in for the reference's ``pipelines/context.py`` (same names, same
results, bit-exact integers).

Reference: ``uniform`` pipelines/context.py:30-59, ``ordered_halving`` :22-27, ``get_context_scheduler``
:62-66, ``compute_num_context`` :7-10, ``compute_context_indices`` :13-19.  Host-side integer logic only.
"""
from typing import Callable, Iterator, List, NamedTuple, Optional, Tuple

import numpy as np

__all__ = ["ordered_halving", "uniform", "get_context_scheduler", "compute_num_context",
           "compute_context_indices", "get_total_steps", "window_table", "overlap_plan", "step_frame_ids", "Wavefront",
           "wavefront_schedule"]


def compute_num_context(init_video_length: int, context_size: int, context_overlap: int) -> int:
    stride = context_size - context_overlap
    return (init_video_length - context_size) // stride + 1


def compute_context_indices(num_context: int, context_size: int, context_overlap: int):
    stride = context_size - context_overlap
    return [(i * stride, i * stride + context_size - 1) for i in range(num_context)]


def ordered_halving(val: int) -> float:
    """Radical inverse in base 2 of a 64-bit integer (van der Corput), in [0, 1)."""
    v, out = int(val) & ((1 << 64) - 1), 0
    for _ in range(64):
        out = (out << 1) | (v & 1)
        v >>= 1
    return out / (1 << 64)


def uniform(step: int = ..., num_frames: int = ..., context_size: Optional[int] = None, context_stride: int = 3,
            context_overlap: int = 4, closed_loop: bool = True) -> Iterator[List[int]]:
    if num_frames <= context_size:
        yield list(range(num_frames))
        return
    n_dilations = min(context_stride, int(np.ceil(np.log2(num_frames / context_size))) + 1)
    frac = ordered_halving(step)
    shift = int(round(num_frames * frac))
    stop = num_frames + shift + (0 if closed_loop else -context_overlap)
    for level in range(n_dilations):
        dilation = 1 << level
        hop = context_size * dilation - context_overlap
        for start in range(int(frac * dilation) + shift, stop, hop):
            frames = []
            for e in range(start, start + context_size * dilation, dilation):
                # indices past the end are reflected back (the reference's `num_frames - 2 - e % num_frames`)
                frames.append(e if e < num_frames else num_frames - 2 - e % num_frames)
            yield frames


def get_context_scheduler(name: str) -> Callable:
    if name == "uniform":
        return uniform
    raise ValueError(f"Unknown context_overlap policy {name}")


def get_total_steps(scheduler, timesteps, num_steps=None, num_frames=..., context_size=None, context_stride=3,
                    context_overlap=4, closed_loop=True):
    return sum(len(list(scheduler(i, num_steps, num_frames, context_size, context_stride, context_overlap)))
               for i in range(len(timesteps)))


def window_table(video_length: int, context_frames: int, context_overlap: int, schedule: str = "uniform"):
    """The call the pipeline makes (reference pipelines/v_express_pipeline.py:486-500): windows for step 0 and
    the per-frame cover count.  The count reproduces the reference's NON-accumulating index-put: a frame that
    appears twice inside one (reflected) window is counted once for that window."""
    windows = list(get_context_scheduler(schedule)(step=0, num_frames=video_length, context_size=context_frames,
                                                   context_stride=1, context_overlap=context_overlap,
                                                   closed_loop=False))
    count = np.zeros(video_length, dtype=np.int64)
    for w in windows:
        count[np.unique(np.asarray(w, dtype=np.int64))] += 1
    return windows, count


def _streaming_replay(windows, count):
    """Integer replay of the reference's streaming bookkeeping (pipelines/v_express_pipeline.py :528-529,552-572): per
    window ``context_counter[context] += 1`` is a NON-accumulating index-put (a repeated frame counts once), the Python
    loop then walks the slots in order, starts a frame's sum at its first slot (``noise_preds[f] is None``), adds every
    further slot, and each time ``context_counter[f] == num_frame_context[f]`` holds it hands the current sum to
    ``scheduler.step`` and resets it.

    Returns (final, steps): ``final[f]`` = the (window, slot) list of the sum whose step lands last in frame f, and
    ``steps[w]`` = the ``step_frame_ids`` window w hands to ``scheduler.step``, in order, repeats included."""
    L = len(count)
    counter = [0] * L
    pending = [None] * L
    final = {}
    steps = []
    for wi, win in enumerate(windows):
        for f in set(win):
            counter[f] += 1
        ids = []
        for li, f in enumerate(win):
            if pending[f] is None:
                pending[f] = []
            pending[f].append((wi, li))
            if counter[f] == int(count[f]):
                final[f] = pending[f]
                pending[f] = None
                ids.append(f)
        steps.append(ids)
    return final, steps


def step_frame_ids(windows, count):
    """Per window, the frames the reference hands to ``scheduler.step`` (its ``step_frame_ids``), in order, a frame
    repeated inside a reflected window once per time it is stepped; the step's ``latents[:, :, ids] = ...`` write
    keeps the last.  A frame is stepped only inside its last window, so every frame appears in exactly one list."""
    return _streaming_replay(windows, count)[1]


def overlap_plan(windows, count):
    """Which window slots end up in a frame's noise prediction, for window lists that may repeat a frame inside one
    (reflected) window, from the replay of ``_streaming_replay``: a frame repeated inside its LAST window is stepped
    more than once from the same input latents and the last write wins (index-put on the host tensor).

    Returns ``rounds[w]`` = list of int32 arrays of len(windows[w]): entry = frame index if that slot's prediction is
    accumulated into the frame's final sum, -1 if the reference discards it; every array holds each frame at most
    once, and the arrays of one window are in the reference's summation order."""
    final, _ = _streaming_replay(windows, count)
    keep = set(slot for slots in final.values() for slot in slots)
    rounds = []
    for wi, win in enumerate(windows):
        per_round = []
        seen = {}
        for li, f in enumerate(win):
            if (wi, li) not in keep:
                continue
            r = seen.get(f, 0)
            seen[f] = r + 1
            while len(per_round) <= r:
                per_round.append(np.full(len(win), -1, dtype=np.int32))
            per_round[r][li] = f
        rounds.append(per_round)
    return rounds


class Wavefront(NamedTuple):
    """Work order of ``wavefront_schedule``; every list but ``order`` is indexed like ``order``."""
    reach: int                      # R: largest index distance between two windows that share a frame
    order: List[Tuple[int, int]]    # (window, step) items
    finalised: List[List[int]]      # frames whose step sum is complete after the item: they get their DDIM update
    chunks: List[List[Tuple[int, int]]]   # VAE chunks [start, stop) whose frames are all final after the item
    loads: List[List[int]]          # frames first read by the item (their conditioning must be ready before it)
    releases: List[List[int]]       # frames no later item reads


def wavefront_schedule(windows, num_steps: int, video_length: int, vae_chunk: int) -> Wavefront:
    """Wavefront order of the ``num_steps`` x ``len(windows)`` window forwards of one video.

    A window at step t reads only its frames' latents after step t - 1, so item (w, t) may run once every window u that
    shares a frame with w has run step t - 1 and those frames got their DDIM update.  With R the largest |u - w| over such
    pairs, the key (t R + w, t) orders the items so that
      * (w, t) comes after (u, t - 1) for every u sharing a frame with w (t R + w >= (t - 1) R + u, ties broken by t);
      * within one step a frame's contributions arrive in window order, the order ``overlap_plan``'s slot arrays assume,
        so its step-t sum is complete after its last window and is stepped there -- before any item of step t + 1 reads
        it and after every item of step t has;
      * each item appears once.
    About R (T - 1) + 1 windows are in flight at a time, and the first frames are final after R T (T + 1) / 2 items.

    Chunks are ``vae_chunk`` frames counted from frame 0 (the chunks of ``VExpressPipeline.decode_latents``) and are
    listed in frame order: a chunk whose frames are final before an earlier chunk's waits for it."""
    W, L, T = len(windows), video_length, num_steps
    if W == 0 or T < 1 or vae_chunk < 1:
        raise ValueError(f"wavefront_schedule: {W} windows, {T} steps, vae_chunk {vae_chunk}")
    first, last = [W] * L, [-1] * L
    for wi, win in enumerate(windows):
        for f in win:
            first[f], last[f] = min(first[f], wi), max(last[f], wi)
    if min(last) < 0:
        raise ValueError(f"wavefront_schedule: frames {[f for f in range(L) if last[f] < 0]} are in no window")
    # windows sharing a frame lie within [first[f], last[f]] of that frame
    reach = max(last[f] - first[f] for f in range(L))
    order = sorted(((w, t) for t in range(T) for w in range(W)), key=lambda it: (it[1] * reach + it[0], it[1]))
    pos = {it: i for i, it in enumerate(order)}
    finalised, loads, releases = [[] for _ in order], [[] for _ in order], [[] for _ in order]
    for f in range(L):
        loads[pos[(first[f], 0)]].append(f)
        releases[pos[(last[f], T - 1)]].append(f)
        for t in range(T):
            finalised[pos[(last[f], t)]].append(f)
    chunks = [[] for _ in order]
    ready = -1
    for c0 in range(0, L, vae_chunk):
        c1 = min(c0 + vae_chunk, L)
        ready = max(ready, max(pos[(last[f], T - 1)] for f in range(c0, c1)))
        chunks[ready].append((c0, c1))
    return Wavefront(reach, order, finalised, chunks, loads, releases)
