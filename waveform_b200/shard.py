"""Multi-GPU plumbing for the spectrum path: one process per GPU, streams sharded contiguously, no data-path
collective (SURVEY.md §8e).  The only exchange is the optional cross-channel peak normalisation
(BASELINE.json configs[4]): a MAX all-reduce of n_frames floats over torch.distributed (NCCL on GPUs, gloo in the
CPU tests), followed by the local wf_peak_normalize pass, or by one wf_render pass when display outputs are wanted.

Nothing here computes spectra; it only decides which rank owns which streams and moves the peak vector.
"""
from __future__ import annotations


def shard_streams(n_streams: int, rank: int, world: int) -> tuple[int, int]:
    """Contiguous block of streams for `rank`: (first, count).  All frames of a stream stay on one GPU so the EMA
    recurrence (src/source_generic.cpp:124-132) and the stereo pair of a source never cross devices."""
    if not (0 <= rank < world):
        raise ValueError("rank out of range")
    base, rem = divmod(n_streams, world)
    count = base + (1 if rank < rem else 0)
    first = rank * base + min(rank, rem)
    return first, count


def allreduce_peak(peak, group=None):
    """In-place MAX all-reduce of the per-frame peak vector (torch tensor on the rank's device)."""
    import torch.distributed as dist

    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(peak, op=dist.ReduceOp.MAX, group=group)
    return peak


def peak_gain(peak, target_db: float, max_gain: float):
    """gain[t] = min(target - peak[t], max_gain): the volume-normalisation rule of src/source_generic.cpp:163 with the
    RMS replaced by the all-reduced peak.  Works on torch tensors and numpy arrays."""
    g = target_db - peak
    return g.clamp(max=max_gain) if hasattr(g, "clamp") else g.clip(max=max_gain)


class ShardedEngine:
    """The rank-local engine plus the cross-GPU peak normalisation step."""

    def __init__(self, engine, group=None):
        self.engine = engine
        self.group = group

    def process_normalized(self, pcm, n_frames, hop, target_db=-3.0, max_gain=30.0, **kw):
        out = self.engine.process(pcm, n_frames, hop, want_peak=True, **kw)
        allreduce_peak(out["peak"], self.group)
        key = "db" if "db" in out else "points"
        self.engine.peak_normalize(out[key], out["peak"], target_db, max_gain)
        return out

    def process_normalized_display(self, pcm, n_frames, hop, target_db=-3.0, max_gain=30.0, want_points=False,
                                   want_pixels=False, **kw):
        """Config 5 with display outputs: the spectrum call (dB rows and peak, no display outputs), the all-reduce, then
        one wf_render pass that normalises the rows in place and renders points / pixels / min from the normalised rows —
        what render() draws from normalised m_decibels."""
        out = self.engine.process(pcm, n_frames, hop, want_peak=True, **kw)
        allreduce_peak(out["peak"], self.group)
        out.update(self.engine.render(out["db"], out["peak"], target_db, max_gain, write_db=True, want_points=want_points,
                                      want_pixels=want_pixels))
        return out
