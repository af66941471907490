"""A context's growable buffers after a failed grow: the call that could not allocate raises E_NOMEM, leaves nothing
behind that a later call or the context's destruction trips over, and the context keeps working.

simplify_spectrum grows its row buffer R[in_height][out_width] before it launches anything, so a thumbnail too large for
the device fails in that grow alone. Every tensor is allocated before the first call: a caching-allocator block placed
on an address the context freed would hide a stale pointer."""
import ctypes

import numpy as np
import pytest

E_NOMEM = -5
IN_HEIGHT = 1 << 20  # channels of one time sample: the row buffer holds 4 * IN_HEIGHT bytes per output column
SMALL_W = 16  # 64 MiB of rows
HUGE_W = 1 << 18  # 1 TiB of rows


@pytest.mark.gpu
def test_failed_grow_leaves_context_usable():
    torch = pytest.importorskip("torch")
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import srtb_b200
    torch.cuda.set_device(0)
    ctx = srtb_b200.Context(0, torch.cuda.current_stream().cuda_stream)
    cudart = ctypes.CDLL("libcudart.so.12")  # the runtime libsrtb_b200 loaded: its last-error state
    cudart.cudaGetLastError()  # whatever an earlier test left there
    try:
        g = torch.Generator(device="cuda").manual_seed(7)
        spec = torch.randn((IN_HEIGHT, 2), generator=g, device="cuda", dtype=torch.float32)  # complex64 [C][1], 8 MiB
        outs = [(torch.empty((1, w), dtype=torch.float32, device="cuda"),
                 torch.empty((1, w), dtype=torch.int32, device="cuda"),
                 torch.empty(1, dtype=torch.float32, device="cuda")) for w in (SMALL_W, HUGE_W, SMALL_W)]
        torch.cuda.synchronize()

        def call(width, out):
            ctx.simplify_spectrum(spec, 1, IN_HEIGHT, width, 1, *out)
            torch.cuda.synchronize()

        call(SMALL_W, outs[0])
        first = [t.cpu().numpy().copy() for t in outs[0]]

        if torch.cuda.get_device_properties(0).total_memory >= 4 * IN_HEIGHT * HUGE_W:
            pytest.skip("the device could hold the oversized row buffer")
        with pytest.raises(srtb_b200.SrtbError) as ei:
            call(HUGE_W, outs[1])
        assert ei.value.code == E_NOMEM, ei.value

        call(SMALL_W, outs[2])
        for a, b in zip(first, (t.cpu().numpy() for t in outs[2])):
            assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    finally:
        ctx.close()
    torch.cuda.synchronize()
    assert cudart.cudaGetLastError() == 0
