"""The host-thread harness of the native batch entry points (ygz_vo_run_stages, ygz_vo_run_ex, ygz_vo_run_handoff_ex):
how the streams are split over host threads and where the timed region starts change no result and no transfer count.

Setting of test_vo.test_native_driver_matches_python_loop: 3 sliding-crop streams of 26 frames, key-frame policy 5 / 0.03 /
0.03.  Every stream's windows and key-frame jobs are decided by that stream alone, so a run on 1, 2 or 3 host threads
(each with its own context) gives the same trajectories and counters bit for bit, and so does a run whose warm-up ends at
another frame.  A hand-over already equals a run split at warm = handoff (test_map_record, test_reference_record); here it
must not depend on the thread split either."""
import numpy as np
import pytest

from ygz_slam_b200 import synth

N_STREAMS, N_FRAMES, WARM, HANDOFF = 3, 26, 13, 11
POLICY = (5, 0.03, 0.03)
THREADS = (1, 2, 3)
IMAGE_BYTES = 640 * 480
# name -> vo_native.run keywords
CONFIGS = {
    "stages": dict(engine="stages"),
    "resident_w1_keyframe": dict(window=1, ref_mode="keyframe"),
    "resident_w1_previous": dict(window=1, ref_mode="previous"),
    "resident_w8_keyframe": dict(window=8, ref_mode="keyframe"),
    "resident_w8_previous": dict(window=8, ref_mode="previous"),
    "handoff_keyframe": dict(window=8, ref_mode="keyframe", handoff=HANDOFF),
    "handoff_previous": dict(window=8, ref_mode="previous", handoff=HANDOFF),
}


@pytest.fixture(scope="module")
def batch():
    from ygz_slam_b200 import vo_native
    data = [synth.shift_stream(s, N_FRAMES) for s in range(N_STREAMS)]
    return vo_native.stack_pinned([d[0] for d in data]), [d[1] for d in data]


@pytest.fixture(scope="module")
def runs(ctx3, batch):
    """(config, threads, warm) -> (trajectory, stats, seconds, details); hand-overs run at warm = handoff only."""
    from ygz_slam_b200 import vo_native
    frames, depths = batch
    out = {}
    for name, kw in CONFIGS.items():
        warms = (HANDOFF,) if "handoff" in kw else (0, WARM)
        for warm in warms:
            for threads in (THREADS if warm == warms[0] else (1,)):
                out[name, threads, warm] = vo_native.run(ctx3, frames, depths, *POLICY, warm=warm, threads=threads, details=True, **kw)
    return out


def _warms(name):
    return (HANDOFF,) if "handoff" in CONFIGS[name] else (0, WARM)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CONFIGS))
def test_thread_split_changes_no_result(runs, name):
    warm = _warms(name)[0]
    traj, stats, _, _ = runs[name, 1, warm]
    assert all(not s["lost"] and s["keyframes"] >= 3 and s["ba"] >= 2 for s in stats), stats
    for threads in THREADS[1:]:
        traj_t, stats_t, _, _ = runs[name, threads, warm]
        assert np.array_equal(traj, traj_t), threads
        assert stats == stats_t, threads


@pytest.mark.gpu
@pytest.mark.parametrize("name", [n for n in CONFIGS if "handoff" not in CONFIGS[n]])
def test_warm_up_only_moves_the_timed_region(runs, name):
    traj, stats, _, _ = runs[name, 1, 0]
    traj_w, stats_w, _, _ = runs[name, 1, WARM]
    assert np.array_equal(traj, traj_w)
    assert stats == stats_w


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CONFIGS))
def test_timed_region_details(runs, name):
    for key, (_, _, sec, det) in runs.items():
        if key[0] != name:
            continue
        assert sec > 0 and det["device_ms"] > 0 and det["gpu_launches"] > 0, (key, sec, det)


@pytest.mark.gpu
def test_stages_upload_every_timed_frame_once(runs):
    for (name, threads, warm), (*_, det) in runs.items():
        if name == "stages":
            assert det["h2d_image_bytes"] == N_STREAMS * (N_FRAMES - warm) * IMAGE_BYTES, (threads, warm)


@pytest.mark.gpu
@pytest.mark.parametrize("name", [n for n in CONFIGS if n != "stages"])
def test_resident_transfers_do_not_depend_on_the_thread_split(runs, name):
    warm = _warms(name)[0]
    keys = ("h2d_image_bytes", "h2d_other_bytes", "d2h_bytes")
    want = [runs[name, 1, warm][3][k] for k in keys]
    assert want[0] > 0 and want[1] > 0 and want[2] > 0
    for threads in THREADS[1:]:
        assert [runs[name, threads, warm][3][k] for k in keys] == want, threads
