"""Compile the REFERENCE's own LocalConv CUDA kernels to sm_90a cubins under oracle/_ref/.  TEST INFRASTRUCTURE ONLY.

    python -m oracle.build_ref_kernels            # needs /root/reference (build container); writes oracle/_ref/

The reference keeps its kernels as C source strings inside Python (cupy_layers/aggregation_zeropad.py:20-110,
aggregation_zeropad_mix.py:20-207), substitutes every dimension as a literal (cupy_layers/utils.py:14-18,
`Template(code).substitute(**kwargs)`) and compiles them through CuPy/NVRTC at first use.  CuPy is absent here and
/root/reference does not exist on the GPU box, so this recipe performs exactly that build step ahead of time:

  * the reference module is imported unmodified (oracle/ref_import.py shims `cupy`);
  * `cupy.cuda.compile_with_cache` is pointed at nvcc (`-cubin -arch=sm_90a`), and the reference's OWN
    `load_kernel(name, code, **literals)` is called with the literals its forward/backward pass for a shape
    (aggregation_zeropad.py:130-139,155-163,170,179; mix :230-241,257-269,274,284);
  * only BINARY outputs land in oracle/_ref/ (one cubin per kernel x shape x dtype + manifest.json with the launch
    geometry the reference uses: block (1024,1,1), grid (GET_BLOCKS(n),1,1), :14-18,140-143).  No reference source is
    copied into the repository; oracle/_ref/ is git-ignored and travels to the GPU box with the snapshot.

tests/test_ref_kernels_gpu.py launches these cubins with the driver API on the same inputs as libcotb200 (parity against
the reference's real GPU kernels, the bar BASELINE.json states); tools/bench_ref_kernels.py times them beside ours.
"""
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "oracle", "_ref")

# (tag, N, C, H, W, heads, wc, k, pad) -- stride 1, dilation 1 everywhere (the only use in the model zoo)
AGG_SHAPES = [
    ("cfg1", 2, 64, 32, 32, 1, 8, 3, 1),            # BASELINE.json configs[0]
    ("selftest_k5", 2, 8, 9, 9, 2, 4, 5, 2),        # aggregation_zeropad.py:238-265
    ("selftest_k1", 2, 8, 9, 9, 2, 4, 1, 0),        # :267-292
    ("ragged", 3, 24, 7, 5, 1, 3, 3, 1),
    ("s1_b8", 8, 64, 56, 56, 1, 8, 3, 1),
    ("s1_b256", 256, 64, 56, 56, 1, 8, 3, 1),       # CoTNet-50 bs256 stage shapes (SURVEY.md 8d)
    ("s2_b256", 256, 128, 28, 28, 1, 16, 3, 1),
    ("s3_b256", 256, 256, 14, 14, 1, 32, 3, 1),
    ("s4_b256", 256, 512, 7, 7, 1, 64, 3, 1),
]
AGG_DTYPES = {"cfg1": ("float", "double"), "selftest_k5": ("double",), "selftest_k1": ("double",), "ragged": ("float", "double")}
# mix: (tag, N, C, H, W, heads, wc) with k1=3/pad 1, k2=5/pad 2 (aggregation_zeropad_mix.py:344-349)
MIX_SHAPES = [("mix_selftest", 2, 8, 6, 6, 1, 4), ("mix_s1_b32", 32, 64, 56, 56, 1, 8)]
# the other cupy_layers variants (SURVEY 8f rank 4): (tag, N, C, H, W, heads, wc[, k, pad])
REFPAD_SHAPES = [("refpad_selftest", 2, 8, 9, 9, 2, 4, 5, 2),     # aggregation_refpad.py:225-233
                 ("refpad_k3", 3, 24, 14, 10, 1, 3, 3, 1), ("refpad_s2_b8", 8, 128, 28, 28, 1, 16, 3, 1)]
DILATE_SHAPES = [("dilate_selftest", 2, 8, 7, 7, 2, 4),           # aggregation_zeropad_dilate.py:258-264
                 ("dilate_s2_b8", 8, 128, 28, 28, 1, 16)]
MERGE_SHAPES = [("merge_selftest", 2, 8, 6, 6, 2, 4),             # aggregation_zeropad_mix_merge.py:332-339
                ("merge_s1_b8", 8, 64, 56, 56, 1, 8)]


class _NvccModule:
    def __init__(self, cubin):
        self.cubin = cubin

    def get_function(self, name):
        return (name, self.cubin)


def _compile_with_cache(code):
    """Stand-in for cupy.cuda.compile_with_cache: same input (the substituted source), nvcc instead of NVRTC."""
    with tempfile.TemporaryDirectory() as td:            # the source text never touches the repository
        src, dst = os.path.join(td, "k.cu"), os.path.join(td, "k.cubin")
        open(src, "w").write(code)
        subprocess.run(["nvcc", "-cubin", "-arch=sm_90a", "-O3", "-o", dst, src], check=True, capture_output=True)
        return _NvccModule(open(dst, "rb").read())


def main():
    from oracle import ref_import
    if not ref_import.available():
        print("oracle/build_ref_kernels: no reference tree at %s; keeping whatever is in oracle/_ref/" % ref_import.REF)
        return 0
    ns = ref_import.load()
    import cupy
    cupy.cuda.compile_with_cache = _compile_with_cache
    sys.path.insert(0, ref_import.REF)
    import cupy_layers.utils as ref_utils
    import cupy_layers.aggregation_zeropad_mix as ref_mix
    ref_agg = ns.agg_module
    os.makedirs(OUT, exist_ok=True)
    manifest = {"block": ref_agg.CUDA_NUM_THREADS, "kernels": []}

    def emit(tag, name, code, nthreads, lit, meta, grid_n=None):
        fn, cubin = ref_utils.load_kernel(name, code, nthreads=nthreads, **lit)
        fname = "%s__%s__%s.cubin" % (name, tag, lit["Dtype"])
        open(os.path.join(OUT, fname), "wb").write(cubin)
        manifest["kernels"].append(dict(meta, tag=tag, kernel=fn, file=fname, dtype=lit["Dtype"], nthreads=nthreads,
                                        grid=ref_agg.GET_BLOCKS(grid_n if grid_n is not None else nthreads)))

    for tag, N, C, H, W, heads, wc, k, pad in AGG_SHAPES:
        Ho, Wo = H + 2 * pad - k + 1, W + 2 * pad - k + 1
        for dt in AGG_DTYPES.get(tag, ("float",)):
            lit = dict(Dtype=dt, num=N, input_channels=C, weight_heads=heads, weight_channels=wc, bottom_height=H,
                       bottom_width=W, top_height=Ho, top_width=Wo, kernel_h=k, kernel_w=k, stride_h=1, stride_w=1,
                       dilation_h=1, dilation_w=1, pad_h=pad, pad_w=pad)
            meta = dict(op="agg", N=N, C=C, H=H, W=W, heads=heads, wc=wc, k=k, pad=pad, Ho=Ho, Wo=Wo)
            emit(tag, "aggregation_zeropad_forward_kernel", ref_agg._aggregation_zeropad_forward_kernel,
                 N * heads * C * Ho * Wo, lit, meta)                                           # :124,130
            emit(tag, "aggregation_zeropad_input_backward_kernel", ref_agg._aggregation_zeropad_input_backward_kernel,
                 N * C * H * W, lit, meta)                                                     # :170-172
            emit(tag, "aggregation_zeropad_weight_backward_kernel", ref_agg._aggregation_zeropad_weight_backward_kernel,
                 N * heads * wc * Ho * Wo, lit, meta)                                          # :179-181
    for tag, N, C, H, W, heads, wc in MIX_SHAPES:
        for dt in (("double", "float") if tag == "mix_selftest" else ("float",)):
            lit = dict(Dtype=dt, num=N, input_channels=C, weight_heads=heads, weight_channels=wc, bottom_height=H,
                       bottom_width=W, top_height=H, top_width=W, kernel1_h=3, kernel1_w=3, kernel2_h=5, kernel2_w=5,
                       stride_h=1, stride_w=1, dilation_h=1, dilation_w=1, pad1_h=1, pad1_w=1, pad2_h=2, pad2_w=2)
            meta = dict(op="mix", N=N, C=C, H=H, W=W, heads=heads, wc=wc)
            emit(tag, "aggregation_zeropad_mix_forward_kernel", ref_mix._aggregation_zeropad_mix_forward_kernel,
                 N * 2 * heads * C * H * W, lit, meta)                                         # mix :220-221
            emit(tag, "aggregation_zeropad_mix_input_backward_kernel", ref_mix._aggregation_zeropad_mix_input_backward_kernel,
                 N * C * H * W, lit, meta)                                                     # :273-274
            emit(tag, "aggregation_zeropad_mix_weight_backward_kernel", ref_mix._aggregation_zeropad_mix_weight_backward_kernel,
                 2 * N * heads * wc * H * W, lit, meta, grid_n=N * heads * wc * H * W)         # :283-284 (grid from n, loop to 2n)
    import cupy_layers.aggregation_refpad as ref_refpad
    import cupy_layers.aggregation_zeropad_dilate as ref_dilate
    import cupy_layers.aggregation_zeropad_mix_merge as ref_merge
    for tag, N, C, H, W, heads, wc, k, pad in REFPAD_SHAPES:
        Ho, Wo = H + 2 * pad - k + 1, W + 2 * pad - k + 1
        for dt in (("double", "float") if "selftest" in tag or tag == "refpad_k3" else ("float",)):
            lit = dict(Dtype=dt, num=N, input_channels=C, weight_heads=heads, weight_channels=wc, bottom_height=H,
                       bottom_width=W, top_height=Ho, top_width=Wo, kernel_h=k, kernel_w=k, stride_h=1, stride_w=1,
                       dilation_h=1, dilation_w=1, pad_h=pad, pad_w=pad)
            meta = dict(op="refpad", N=N, C=C, H=H, W=W, heads=heads, wc=wc, k=k, pad=pad, Ho=Ho, Wo=Wo)
            emit(tag, "aggregation_refpad_forward_kernel", ref_refpad._aggregation_refpad_forward_kernel,
                 N * heads * C * Ho * Wo, lit, meta)                                           # refpad :141-142
            emit(tag, "aggregation_refpad_input_backward_kernel", ref_refpad._aggregation_refpad_input_backward_kernel,
                 N * C * (H + 2 * pad) * (W + 2 * pad), lit, meta)                             # :185-187 (padded grid)
            emit(tag, "aggregation_refpad_weight_backward_kernel", ref_refpad._aggregation_refpad_weight_backward_kernel,
                 N * heads * wc * Ho * Wo, lit, meta)                                          # :203-205
    for tag, N, C, H, W, heads, wc in DILATE_SHAPES:
        for dt in (("double", "float") if "selftest" in tag else ("float",)):
            lit = dict(Dtype=dt, num=N, input_channels=C, weight_heads=heads, weight_channels=wc, bottom_height=H,
                       bottom_width=W, top_height=H, top_width=W, kernel_h=3, kernel_w=3, stride_h=1, stride_w=1)
            meta = dict(op="dilate", N=N, C=C, H=H, W=W, heads=heads, wc=wc)
            emit(tag, "aggregation_zeropad_dilate_forward_kernel", ref_dilate._aggregation_zeropad_dilate_forward_kernel,
                 N * heads * C * H * W, lit, meta)                                             # dilate :159-160
            emit(tag, "aggregation_zeropad_dilate_input_backward_kernel", ref_dilate._aggregation_zeropad_dilate_input_backward_kernel,
                 N * C * H * W, lit, meta)                                                     # :203-205
            emit(tag, "aggregation_zeropad_dilate_weight_backward_kernel", ref_dilate._aggregation_zeropad_dilate_weight_backward_kernel,
                 N * heads * wc * H * W, lit, meta)                                            # :212-214
    for tag, N, C, H, W, heads, wc in MERGE_SHAPES:
        for dt in (("double", "float") if "selftest" in tag else ("float",)):
            lit = dict(Dtype=dt, num=N, input_channels=C, weight_heads=heads, weight_channels=wc, bottom_height=H,
                       bottom_width=W, top_height=H, top_width=W, kernel1_h=3, kernel1_w=3, kernel2_h=5, kernel2_w=5,
                       stride_h=1, stride_w=1, dilation_h=1, dilation_w=1, pad1_h=1, pad1_w=1, pad2_h=2, pad2_w=2)
            meta = dict(op="merge", N=N, C=C, H=H, W=W, heads=heads, wc=wc)
            emit(tag, "aggregation_zeropad_mix_merge_forward_kernel", ref_merge._aggregation_zeropad_mix_merge_forward_kernel,
                 N * 2 * heads * C * H * W, lit, meta)                                         # merge :196-197
            emit(tag, "aggregation_zeropad_mix_merge_input_backward_kernel", ref_merge._aggregation_zeropad_mix_merge_input_backward_kernel,
                 N * C * H * W, lit, meta)                                                     # :253-255
            emit(tag, "aggregation_zeropad_mix_merge_weight_backward_kernel", ref_merge._aggregation_zeropad_mix_merge_weight_backward_kernel,
                 2 * N * heads * wc * H * W,
                 lit, meta)      # the kernel's own index space (2 kernels x N x heads x wc x Ho x Wo).  The reference's host code
            # derives nthreads from weight.shape[3] of the 4-D packed weight (= Wo, :262), which over- or under-covers it.
    json.dump(manifest, open(os.path.join(OUT, "manifest.json"), "w"), indent=1)
    print("oracle/_ref: %d cubins" % len(manifest["kernels"]))
    return 0


if __name__ == "__main__":
    sys.exit(main())
