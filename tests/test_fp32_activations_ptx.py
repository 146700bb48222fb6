"""The fp32 instantiations of the cell kernels (csrc/lstm_pointwise.cu), of the attention scores (csrc/seq_pool.cu) and of the
heads' generic softmax (csrc/head_xent.cu, csrc/head_wgmma.cu) must not use the approximate activations.  build.py compiles
with --use_fast_math, under which tanhf becomes tanh.approx.f32 and expf / logf / division ex2.approx / lg2.approx / rcp.approx
(relative error up to about 2^-11): the fp32 path would then be no more accurate than the bf16 one, which keeps them on
purpose.  This compiles the files to PTX with the build's own flags and reads every kernel entry; it needs nvcc, not a GPU."""
import os
import re
import shutil
import subprocess

import pytest

from lstm_tensorspark_b200 import build


def _nvcc():
    n = build._nvcc()
    return n if os.path.exists(n) or shutil.which(n) else None


def _entries(src, tmp_path):
    """{mangled kernel name: PTX body} of ``csrc/<src>`` compiled with build.NVCC_FLAGS (as PTX for compute_90a)."""
    flags = [f for f in build.NVCC_FLAGS if f not in build.ARCH_FLAGS]
    i = flags.index("-Xptxas")
    del flags[i:i + 2]                                   # (ptxas options: no ptxas here)
    out = tmp_path / (src + ".ptx")
    subprocess.run([build._nvcc(), "--ptx", *flags, "-gencode", "arch=compute_90a,code=compute_90a", "-o", str(out),
                    os.path.join(build.CSRC, src)], check=True, capture_output=True, text=True)
    bodies = re.split(r"(?m)^\.(?:visible \.)?entry ", out.read_text())[1:]
    return {b.split("(", 1)[0]: b for b in bodies}


@pytest.mark.skipif(_nvcc() is None, reason="needs nvcc")
def test_fp32_cell_kernels_use_no_approximate_activation(tmp_path):
    ents = _entries("lstm_pointwise.cu", tmp_path)
    cells = {n: b for n, b in ents.items() if re.search(r"lstm_pointwise_(fwd|bwd)_kernel", n)}
    assert len(cells) == 8, sorted(cells)               # {fwd, bwd} x {bf16, fp32} x {masked, not}
    fp32 = {n: b for n, b in cells.items() if re.search(r"kernelIfLb0E", n)}
    assert len(fp32) == 4, sorted(cells)
    for n, b in fp32.items():
        # no approximate fp32 tanh or division (sigmoid's 1 / (1 + e^-x)); the fp64 exp and tanh the kernels call instead take
        # a seed from ex2.approx.f32 / rcp.approx.f64 and refine it to fp64 accuracy, so those two may appear
        bad = re.findall(r"\b(?:tanh|rcp|div)\.approx(?:\.ftz)?\.f32", b)
        assert not bad, (n, bad)
    for n, b in cells.items():                           # the bf16 instantiations keep tanh.approx (the control of the parser)
        if n not in fp32:
            assert "tanh.approx.f32" in b, n


@pytest.mark.skipif(_nvcc() is None, reason="needs nvcc")
def test_fp32_attention_scores_use_no_approximate_tanh(tmp_path):
    """Attention pooling's u = tanh(h W_a + b_a): exact in the fp32 instantiation, tanh.approx in the bf16 one."""
    ents = _entries("seq_pool.cu", tmp_path)
    scores = {n: b for n, b in ents.items() if "attn_scores_kernel" in n}
    exact = [n for n in scores if "attn_scores_kernelILb1E" in n]
    fast = [n for n in scores if "attn_scores_kernelILb0E" in n]
    assert len(exact) == 1 and len(fast) == 1, sorted(scores)
    assert "tanh.approx" not in scores[exact[0]]
    assert "tanh.approx.f32" in scores[fast[0]]


@pytest.mark.skipif(_nvcc() is None, reason="needs nvcc")
@pytest.mark.parametrize("src,kernel", [("head_xent.cu", "xent_rows_kernel"), ("head_wgmma.cu", "xent_steps_kernel")])
def test_fp32_softmax_heads_use_no_approximate_exp_or_log(tmp_path, src, kernel):
    """The generic softmax of the last-state and per-step heads: the fp32 instantiation (kExact) takes exp and log in fp64, the
    bf16 one keeps ex2.approx / lg2.approx (the control of the parser)."""
    ents = _entries(src, tmp_path)
    exact = [b for n, b in ents.items() if f"{kernel}ILb1E" in n]
    fast = [b for n, b in ents.items() if f"{kernel}ILb0E" in n]
    assert len(exact) == 1 and len(fast) == 1, sorted(ents)
    assert not re.findall(r"\b(?:ex2|lg2)\.approx(?:\.ftz)?\.f32", exact[0])
    assert re.search(r"\bex2\.approx(?:\.ftz)?\.f32", fast[0]) and re.search(r"\blg2\.approx(?:\.ftz)?\.f32", fast[0])
