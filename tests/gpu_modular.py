"""Decoding Modular files through ModularBatch, for the GPU tests."""
import pytest

from jxl_rs_b200 import abi


def gpu_decode(ctx, files, lanes=1, lz77_stats=False, expect_error=False, refused=(), walk_stats=False):
    """Decodes `files` as one ModularBatch with `lanes` lanes per warp into pinned host buffers. Returns the u8 outputs
    and the i32 planes of the frames the batch kept, then, when asked for, the batch's lz77_stats() before run(), its
    walk_stats() before run() and the JxgError of wait() (None if it succeeded; without `expect_error` the error is raised). Adding a frame whose
    index is in `refused` must raise JxgError; the batch goes on without it."""
    import torch
    import jxl_rs_b200 as j
    frames = [j.ModularParsedFrame(f) for f in files]
    outs = [torch.empty((fr.height, fr.width, 3), dtype=torch.uint8).pin_memory() for fr in frames]
    b = j.ModularBatch(ctx, lanes)
    err = None
    kept = []
    try:
        for i, (fr, o) in enumerate(zip(frames, outs)):
            if i in refused:
                with pytest.raises(abi.JxgError):
                    b.add(fr, o.data_ptr(), fr.width * 3, False)
            else:
                b.add(fr, o.data_ptr(), fr.width * 3, False)
                kept.append(i)
        stats = b.lz77_stats()
        walks = b.walk_stats()
        b.run()
        try:
            b.wait()
        except abi.JxgError as e:
            if not expect_error:
                raise
            err = e
        planes = [b.read_planes(k) for k in range(len(kept))]
    finally:
        b.close()
    result = ([outs[i].numpy().copy() for i in kept], planes)
    if lz77_stats:
        result += (stats,)
    if walk_stats:
        result += (walks,)
    if expect_error:
        result += (err,)
    return result
