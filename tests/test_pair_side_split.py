"""How the pipelined pair's forward side GEMMs share the SMs L_a leaves free (ops/cuda_lstm.py pipelined_fwd_split): pure host
logic, no GPU needed."""
from lstm_tensorspark_b200.ops import cuda_lstm as CL


def test_headline_split_on_an_h100():
    # 132 SMs, L_a holds 64 at H = 1024; gx_a (D = 1024) and gx_b (H_b = 1024) do the same work per step
    assert CL.pipelined_fwd_split(132, 1024, 1024, 1024) == (34, 34)


def test_split_follows_the_work_ratio_and_uses_every_free_sm():
    for sms, d, ha, hb in ((132, 256, 512, 256), (132, 64, 1024, 1024), (132, 4096, 1024, 256), (148, 1024, 1024, 512)):
        n_a, n_b = CL.pipelined_fwd_split(sms, d, ha, hb)
        free = sms - ha // 16
        assert n_a >= 1 and n_b >= 1 and n_a + n_b == free, (sms, d, ha, hb, n_a, n_b)
        assert abs(n_a / free - d / (d + hb)) <= 1 / free, (sms, d, ha, hb, n_a, n_b)


def test_input_projection_before_the_recurrence_leaves_every_free_sm_to_gx_b():
    assert CL.pipelined_fwd_split(132, 0, 1024, 1024) == (0, 68)
