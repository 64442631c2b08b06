"""The kernels a call launches, as torch.profiler records them: shared by the plan routing tests."""
import torch


def check_launches(fn, want):
    """One call of fn launches the CUDA kernels `want`, in order.  A first call plans outside the profiled region.  The profiled
    region runs three calls, and the last two must each launch exactly `want`: a trace can miss the kernels launched just after
    it starts, so the first call only warms it up.  The order is that of the kernels' correlation ids (FunctionEvent.id), which rise
    with the launch calls on the host: with programmatic dependent launch a kernel can start before its predecessor in the stream
    ends, so start times need not follow launch order.  Now and then torch.profiler hands back a trace with no kernel at all
    (seen on an H100 with torch 2.11, in a few captures of a hundred); every plan launches kernels, so such a capture is taken
    again, up to three times, and the first capture holding kernels is compared."""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    for _ in range(3):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(3):
                fn()
            torch.cuda.synchronize()
        evs = [e for e in prof.events() if e.device_type == DeviceType.CUDA and not e.name.startswith(("Memcpy", "Memset"))]
        if evs:
            break
    assert len({e.id for e in evs}) == len(evs), "kernel events without distinct correlation ids"
    names = [e.name for e in sorted(evs, key=lambda e: e.id)]
    assert len(want) > 0 and names[-2 * len(want):] == want + want
