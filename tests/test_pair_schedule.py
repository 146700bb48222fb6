"""How two stacked layers are scheduled (ops/cuda_lstm.py pair_schedule): pure host logic, no GPU needed."""
from lstm_tensorspark_b200.ops import cuda_lstm as CL


def test_pair_schedule_by_device_size():
    T, B, D = 128, 256, 1024
    # H100 SXM: 132 SMs, 120 backward CTAs co-resident in clusters of 4; 64 + 64 + 8 CTAs do not fit side by side
    assert CL.pair_schedule(T, B, D, 1024, 1024, 132, 120) == "pipelined"
    assert CL.pair_schedule(T, B, D, 1024, 1024, 148, 144) == "wavefront"
    assert CL.pair_schedule(T, B, D, 512, 256, 132, 120) == "wavefront"
    assert CL.pair_schedule(T, B, D, 1024, 512, 132, 120) == "wavefront"
    assert CL.pair_schedule(T, B, D, 1024, 1024, 70, 68) is None


def test_pair_schedule_rejects_shapes_outside_both_schedules():
    T, B, D = 128, 256, 1024
    for bad in ((T, 128, D, 1024, 1024), (1, B, D, 1024, 1024), (T, B, D, 2048, 1024), (T, B, D, 1024, 320), (T, B, 12, 1024, 1024)):
        assert CL.pair_schedule(*bad, 132, 120) is None, bad
