"""The stream cases of include/centerpose_b200_video.h (tests/test_video_streams_gpu.py): each case names the entry
points it holds on a side stream.  A helper module: it holds no tests and imports without a GPU."""
STREAM_CASES = {
    "ellipse_poly": ("ellipse_poly_batch",),
    "render_plan": ("render_plan_batch",),
}
