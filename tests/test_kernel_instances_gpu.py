"""Every __global__ kernel of libdsmil_b200.so, template instances one by one, is either reached by a case of the
conditioned forward or backward tables (test_conditioned_forward_gpu.py, test_conditioned_backward_gpu.py) or exempt,
with the test file that holds it to its own reference named.

The hot path is a set of template instances picked at run time from C, D, the form of q and the route: k_qmlp_sm90<CT,
DT, DEV, MODELS>, k_attend<CT, J>, k_attend_gb<CT, J>, k_attend_b<CT, NJ>, k_gemv_tn[_rag]<M1>, ...  A case table that
sits at one D leaves most of them without a tight bar, and nothing says so.  Here:

    CPU   the kernels of the built library (cuobjdump -symbols, demangled with cu++filt, both next to the nvcc that
          build.py uses) equal the kernels of KERNELS exactly: an instance added without an entry fails and is named.
    GPU   each conditioned case runs once through its own runner under torch.profiler (CUDA activities); each launches
          every kernel KERNELS credits to it, and together they launch every kernel that is not exempt.

Numbers are not checked here; the conditioned files do that.
"""
from __future__ import annotations

import os
import re
import subprocess

import pytest
import torch

import test_conditioned_backward_gpu as BW
import test_conditioned_forward_gpu as FW

# ------------------------------------------------------------------------------------------------ the table
# kernel (short name, template arguments as integers) -> the conditioned cases that launch it ("fwd:<case>" or
# "bwd:<case>"), or Exempt(test file that holds it to its own reference, why)
class Exempt(str):
    pass


JPEG = Exempt("test_zz_jpeg_gpu.py: the device JPEG decoder, bit for bit against PIL")
NORM = Exempt("test_conditioned_embedder_gpu.py: the InstanceNorm kernels against an fp64 norm on slide-like patches")
EMBED = Exempt("test_embed.py: the u8 HWC -> f32 CHW patch conversion, equal to torchvision's to_tensor")
GATHER = Exempt("test_feed.py: the dropout_patches row gather, equal to indexing")

KERNELS = {
    "k_argmax": ("fwd:tc_d512_c1_n20000_rescale", "fwd:tc_d128_c2_n3000",),
    "k_attend<1,1>": ("fwd:genlin_d166_c1_n3000", "bwd:pv_gen_d166_c1_mask",),
    "k_attend<1,2>": ("fwd:genlin_d512_c1_n2000",),
    "k_attend<1,4>": ("fwd:genlin_d1024_c1_n2000",),
    "k_attend<1,8>": ("fwd:genlin_d1920_c1_n2000",),
    "k_attend<1,16>": ("fwd:tc_d4096_c1_n1500", "bwd:tc_d4096_c1_n1025",),
    "k_attend<2,1>": ("fwd:gen_d166_c2_n2500", "bwd:shard_per_bag_d166",),
    "k_attend<2,2>": ("fwd:gen_d300_c2_n2000", "bwd:bags_d512_misaligned",),
    "k_attend<2,4>": ("fwd:gen_d1000_c2_n2000",),
    "k_attend<2,8>": ("fwd:genlin_d2048_c2_n2000",),
    "k_attend<2,16>": ("fwd:tc_d4096_c2_n1200", "fwd:gen_d2049_c2_n1500",),
    "k_attend<4,1>": ("fwd:genlin_d230_c3_n12000_rescale",),
    "k_attend<4,2>": ("fwd:genlin_d512_c3_n2000",),
    "k_attend<4,4>": ("fwd:gen_d1020_c4_n1500",),
    "k_attend<4,8>": ("fwd:tc_d1152_c3_n1500", "bwd:gen_d1028_c4_n2049",),
    "k_attend<4,16>": ("fwd:tc_d4096_c4_n1000",),
    "k_attend<8,1>": ("fwd:tc_d256_c8_n2000",),
    "k_attend<8,2>": ("fwd:tcgen_d512_c6_n1500", "bwd:tc_d512_c6_n2049", "bwd:tc_d512_c8_n2049",),
    "k_attend<8,4>": ("fwd:tc_d768_c5_n1500",),
    "k_attend<8,8>": ("fwd:tc_d2048_c8_n1000",),
    "k_attend<8,16>": ("fwd:tc_d2944_c8_n1000", "fwd:gen_d3072_c8_n1000", "fwd:gen_d4095_c7_n1000",),
    "k_attend_b<1,1>": ("fwd:tc_d512_c1_n20000_rescale", "fwd:bags_tc_d512_c1", "fwd:models_tc_d512_c1",),
    "k_attend_b<1,2>": ("fwd:bags_tc_d1024_c1", "bwd:bags_d1024_c1",),
    "k_attend_b<1,4>": ("fwd:bags_tc_d2048_c1", "fwd:models_tc_d2048_c1",),
    "k_attend_b<2,1>": ("fwd:tc_d512_c2_n3000", "bwd:shard_bags_d512",),
    "k_attend_b<2,2>": ("fwd:bags_tc_d1024_c2", "fwd:models_tc_d1024_c2",),
    "k_attend_b<2,4>": ("fwd:bags_tc_d2048_c2", "bwd:bags_d2048",),
    "k_attend_b<4,1>": ("fwd:bags_tc_d512_c3", "fwd:models_tc_d512_c3",),
    "k_attend_b<4,2>": ("fwd:tc_d1024_c4_n2000", "bwd:models_d1024_c4",),
    "k_attend_gb<1,1>": ("fwd:bags_genlin_d256_c1", "bwd:bags_gen_d166", "bwd:dev_gen_d166",),
    "k_attend_gb<1,2>": ("fwd:bags_genlin_d512_c1",),
    "k_attend_gb<1,4>": ("fwd:bags_genlin_d1024_c1",),
    "k_attend_gb<1,8>": ("fwd:bags_genlin_d1920_c1",),
    "k_attend_gb<1,16>": ("fwd:bags_tc_d4096_c1",),
    "k_attend_gb<2,1>": ("fwd:bags_genlin_d230_c2", "fwd:bags_gen_d7_c2", "bwd:dev_gen_d230_linear",),
    "k_attend_gb<2,2>": ("fwd:value_tc_d512_c2", "fwd:value_tc_d512_c2_mask",),
    "k_attend_gb<2,4>": ("fwd:bags_gen_d1000_c2",),
    "k_attend_gb<2,8>": ("fwd:value_tc_d2048_c2",),
    "k_attend_gb<2,16>": ("fwd:bags_tc_d2176_c2",),
    "k_attend_gb<4,1>": ("fwd:value_gen_d166_c3_mask",),
    "k_attend_gb<4,2>": ("fwd:bags_genlin_d384_c4",),
    "k_attend_gb<4,4>": ("fwd:bags_gen_d1020_c3",),
    "k_attend_gb<4,8>": ("fwd:bags_tc_d2048_c3", "bwd:bags_gen_d1028_c4",),
    "k_attend_gb<4,16>": ("fwd:bags_tc_d4096_c4",),
    "k_attend_gb<8,1>": ("fwd:bags_gen_d166_c5",),
    "k_attend_gb<8,2>": ("fwd:bags_tc_d512_c6", "bwd:bags_d512_c8",),
    "k_attend_gb<8,4>": ("fwd:bags_gen_d777_c5",),
    "k_attend_gb<8,8>": ("fwd:bags_tc_d1280_c8",),
    "k_attend_gb<8,16>": ("fwd:bags_gen_d4095_c8",),
    "k_axpy_mask": ("bwd:pv_tc_d512_c2", "bwd:pv_gen_d166_c1_mask",),
    "k_bwd_bag": ("bwd:tc_d512_c2_n10000", "bwd:shard_per_bag_d166",),
    "k_bwd_bag_b": ("bwd:bags_d512_rps128", "bwd:shard_bags_d512",),
    "k_bwd_bag_models": ("bwd:models_m2", "bwd:models_d1024_c4",),
    "k_bwd_dL": ("bwd:tc_d512_c2_n10000", "bwd:shard_per_bag_d166",),
    "k_bwd_dL_b": ("bwd:bags_d512_rps128", "bwd:shard_bags_d512",),
    "k_bwd_dL_models": ("bwd:models_m2", "bwd:models_d1024_c4",),
    "k_bwd_dq": ("bwd:tc_d512_c2_n10000", "bwd:shard_per_bag_d166",),
    "k_bwd_dq_b": ("bwd:bags_d512_rps128", "bwd:shard_bags_d512",),
    "k_bwd_dx_extra": ("bwd:tc_d512_c2_n10000", "bwd:tc_d4096_c1_n1025",),
    "k_bwd_dx_extra_b": ("bwd:bags_d512_rps128", "bwd:bags_d512_c8",),
    "k_bwd_dx_extra_models": ("bwd:models_m2", "bwd:models_d1024_c4",),
    "k_bwd_dzv": ("bwd:pv_tc_d512_c2", "bwd:pv_gen_d166_c1_mask",),
    "k_bwd_rowdot_b": ("bwd:bags_d512_rps128", "bwd:shard_bags_d512",),
    "k_bwd_rowdot_models": ("bwd:models_m2", "bwd:models_d1024_c4",),
    "k_bwd_t_partial": ("bwd:tc_d512_c2_n10000", "bwd:shard_per_bag_d166",),
    "k_colsum": ("bwd:tc_d512_c2_n10000", "bwd:shard_per_bag_d166",),
    "k_colsum_rag": ("bwd:models_m2", "bwd:models_d1024_c4",),
    "k_combine_rec": ("fwd:tcgen_d512_c6_n1500", "bwd:shard_per_bag_d166",),
    "k_combine_rec_b": ("fwd:bags_gen_d166_c5", "bwd:dev_gen_d230_linear",),
    "k_crit_qmax_b": ("fwd:bags_gen_d166_c5", "bwd:dev_gen_d230_linear",),
    "k_empty_rec": ("fwd:shard_genlin_d166_c2", "bwd:shard_per_bag_d166",),
    "k_finalize": ("fwd:tcgen_d512_c6_n1500", "bwd:shard_per_bag_d166",),
    "k_finalize_b<0>": ("fwd:tc_d512_c1_n20000_rescale", "bwd:shard_bags_d512",),
    "k_finalize_b<1>": ("fwd:models_tc_d512_c2", "bwd:models_d1024_c4",),
    "k_finalize_gb": ("fwd:bags_gen_d166_c5", "bwd:dev_gen_d230_linear",),
    "k_gather_cand": ("fwd:tcgen_d512_c6_n1500", "bwd:shard_per_bag_d166",),
    "k_gather_cand_b": ("fwd:shard_tc_d512_c2", "bwd:shard_bags_d512",),
    "k_gather_rows": GATHER,
    "k_gemm_tn": ("bwd:tc_d512_c2_n10000", "bwd:shard_per_bag_d166",),
    "k_gemm_tn_rag": ("bwd:bags_d512_rps128", "bwd:shard_bags_d512",),
    "k_gemv_tn<1>": ("bwd:gen_d166_c1_n2049", "bwd:tc_d4096_c1_n1025",),
    "k_gemv_tn<2>": ("bwd:tc_d512_c2_n10000", "bwd:shard_per_bag_d166",),
    "k_gemv_tn<3>": ("bwd:tc_d1024_c3_n2049",),
    "k_gemv_tn<4>": ("bwd:tc_d1024_c4_n2049", "bwd:gen_d1028_c4_n2049",),
    "k_gemv_tn_rag<1>": ("bwd:bags_d1024_c1",),
    "k_gemv_tn_rag<2>": ("bwd:bags_d512_rps128", "bwd:shard_bags_d512",),
    "k_gemv_tn_rag<3>": ("bwd:bags_d1024_c3", "bwd:dev_d1024_c3", "bwd:models_d1024_c3",),
    "k_gemv_tn_rag<4>": ("bwd:bags_d1024_c4", "bwd:dev_d1024_c4", "bwd:models_d1024_c4",),
    "k_instnorm_nhwc": NORM,
    "k_instnorm_plane<0>": NORM,
    "k_instnorm_plane<1>": NORM,
    "k_instnorm_warp": NORM,
    "k_jpeg_color": JPEG,
    "k_jpeg_entropy": JPEG,
    "k_jpeg_idct": JPEG,
    "k_linear<0,0>": ("fwd:genlin_d230_c3_n12000_rescale", "bwd:gen_d230_linear_n2305",),
    "k_linear<0,1>": ("bwd:tc_d512_c2_n10000", "bwd:bags_d512_c8",),
    "k_linear<1,0>": ("fwd:gen_d166_c2_n2500", "bwd:shard_per_bag_d166",),
    "k_linear<2,0>": ("fwd:gen_d166_c2_n2500", "bwd:shard_per_bag_d166",),
    "k_linear<3,1>": ("bwd:tc_d512_c2_n10000", "bwd:shard_per_bag_d166",),
    "k_linear_b<0>": ("fwd:bags_genlin_d230_c2", "bwd:dev_gen_d230_linear",),
    "k_linear_b<1>": ("fwd:bags_gen_d166_c5", "bwd:dev_gen_d166",),
    "k_linear_models<0,1>": ("bwd:models_m2", "bwd:models_d1024_c4",),
    "k_linear_models<3,1>": ("bwd:models_m2", "bwd:models_d1024_c4",),
    "k_merge_cand": ("fwd:tcgen_d512_c6_n1500", "bwd:shard_per_bag_d166",),
    "k_plan_bags": ("fwd:bags_tc_d512_c2", "bwd:shard_bags_d512",),
    "k_plan_bags_gen": ("fwd:bags_gen_d166_c5", "bwd:dev_gen_d230_linear",),
    "k_plan_bags_models": ("fwd:models_tc_d512_c2", "bwd:models_d1024_c4",),
    "k_prep_wimg2": ("fwd:tc_d512_c1_n20000_rescale", "bwd:shard_bags_d512",),
    "k_prep_wimg2_models": ("fwd:models_tc_d512_c2", "bwd:models_d1024_c4",),
    "k_qmlp_sm90<1,0,0,0>": ("fwd:tc_d4096_c1_n1500", "bwd:bags_d1024_c1",),
    "k_qmlp_sm90<1,0,0,1>": ("fwd:models_tc_d1024_c1", "fwd:models_tc_d2048_c1",),
    "k_qmlp_sm90<1,0,1,0>": ("fwd:bags_tc_d1024_c1", "fwd:bags_tc_d4096_c1",),
    "k_qmlp_sm90<1,0,1,1>": ("fwd:models_tc_d1024_c1", "fwd:models_tc_d2048_c1",),
    "k_qmlp_sm90<1,512,0,0>": ("fwd:tc_d512_c1_n20000_rescale", "fwd:bags_tc_d512_c1",),
    "k_qmlp_sm90<1,512,0,1>": ("fwd:models_tc_d512_c1",),
    "k_qmlp_sm90<1,512,1,0>": ("fwd:bags_tc_d512_c1",),
    "k_qmlp_sm90<1,512,1,1>": ("fwd:models_tc_d512_c1",),
    "k_qmlp_sm90<2,0,0,0>": ("fwd:tc_d4096_c2_n1200", "bwd:bags_d2048",),
    "k_qmlp_sm90<2,0,0,1>": ("fwd:models_tc_d1024_c2", "fwd:models_tc_d2048_c2",),
    "k_qmlp_sm90<2,0,1,0>": ("fwd:bags_tc_d1024_c2", "fwd:bags_tc_d2176_c2",),
    "k_qmlp_sm90<2,0,1,1>": ("fwd:models_tc_d1024_c2", "fwd:models_tc_d2048_c2",),
    "k_qmlp_sm90<2,512,0,0>": ("fwd:tc_d512_c2_n3000", "bwd:shard_bags_d512",),
    "k_qmlp_sm90<2,512,0,1>": ("fwd:models_tc_d512_c2", "bwd:models_m2", "bwd:models_m3",),
    "k_qmlp_sm90<2,512,1,0>": ("fwd:bags_tc_d512_c2", "bwd:dev_d512_rps128", "bwd:shard_bags_d512",),
    "k_qmlp_sm90<2,512,1,1>": ("fwd:models_tc_d512_c2", "bwd:models_m2", "bwd:models_m3",),
    "k_qmlp_sm90<4,0,0,0>": ("fwd:tc_d1024_c4_n2000", "bwd:bags_d1024_c4",),
    "k_qmlp_sm90<4,0,0,1>": ("fwd:models_tc_d1024_c4", "bwd:models_d1024_c3", "bwd:models_d1024_c4",),
    "k_qmlp_sm90<4,0,1,0>": ("fwd:bags_tc_d1024_c4", "bwd:dev_d1024_c4",),
    "k_qmlp_sm90<4,0,1,1>": ("fwd:models_tc_d1024_c4", "bwd:models_d1024_c3", "bwd:models_d1024_c4",),
    "k_qmlp_sm90<4,512,0,0>": ("fwd:bags_tc_d512_c3",),
    "k_qmlp_sm90<4,512,0,1>": ("fwd:models_tc_d512_c3",),
    "k_qmlp_sm90<4,512,1,0>": ("fwd:bags_tc_d512_c3",),
    "k_qmlp_sm90<4,512,1,1>": ("fwd:models_tc_d512_c3",),
    "k_qmlp_sm90<8,0,0,0>": ("fwd:tc_d2944_c8_n1000", "fwd:bags_tc_d1280_c8",),
    "k_qmlp_sm90<8,0,1,0>": ("fwd:bags_tc_d1280_c8",),
    "k_qmlp_sm90<8,512,0,0>": ("fwd:tcgen_d512_c6_n1500", "bwd:bags_d512_c8",),
    "k_qmlp_sm90<8,512,1,0>": ("fwd:bags_tc_d512_c6",),
    "k_rowdot": ("bwd:tc_d512_c2_n10000", "bwd:shard_per_bag_d166",),
    "k_scores<0>": ("fwd:gen_d166_c2_n2500", "bwd:shard_per_bag_d166",),
    "k_scores<1>": ("fwd:gen_d300_c2_n2000", "bwd:gen_d1028_c4_n2049",),
    "k_scores<2>": ("fwd:gen_d3072_c8_n1000", "fwd:genlin_d512_c3_n2000",),
    "k_scores_b": ("fwd:bags_gen_d166_c5", "bwd:dev_gen_d230_linear",),
    "k_sum_partials": ("bwd:tc_d512_c2_n10000", "bwd:shard_per_bag_d166",),
    "k_sum_partials_models": ("bwd:models_m2", "bwd:models_d1024_c4",),
    "k_sum_segments": ("bwd:bags_d512_rps128", "bwd:shard_bags_d512",),
    "k_sum_segments_models": ("bwd:models_m2", "bwd:models_d1024_c4",),
    "k_u8hwc_to_f32chw": EMBED,
    "k_vproj_b": ("fwd:value_tc_d512_c2", "fwd:value_tc_d2048_c2",),
}


# ---------------------------------------------------------------------------------------------- name handling
def kernel_key(sym: str) -> str:
    """'void dsmil::sm90::k_qmlp_sm90<(int)1, (int)0, (bool)0, (bool)1>(...)' or the profiler's '... <1, 0, false, true>
    (...)' -> 'k_qmlp_sm90<1,0,0,1>'; a kernel without template arguments keeps its bare name."""
    s = sym.strip()
    if s.startswith("void "):
        s = s[5:]
    depth = 0
    for i, ch in enumerate(s):
        if ch == "<":
            depth += 1
        elif ch == ">":
            depth -= 1
        elif ch == "(" and depth == 0:
            s = s[:i]
            break
    name, _, args = s.partition("<")
    name = name.split("::")[-1]
    if not args:
        return name
    vals = []
    for a in args[:-1].split(","):
        a = re.sub(r"^\((int|bool|unsigned int)\)", "", a.strip())
        vals.append({"true": "1", "false": "0"}.get(a, a))
    return f"{name}<{','.join(vals)}>"


def _toolkit_tools():
    from dsmil_wsi_b200 import build
    bindir = os.path.dirname(os.path.realpath(build._nvcc()))
    tools = [os.path.join(bindir, t) for t in ("cuobjdump", "cu++filt")]
    for t in tools:
        assert os.access(t, os.X_OK), f"{t} is missing: it ships with the toolkit that builds the library"
    return tools


def demangle(names):
    _, filt = _toolkit_tools()
    out = subprocess.run([filt], input="\n".join(names) + "\n", capture_output=True, text=True, check=True).stdout
    dem = out.splitlines()
    assert len(dem) == len(names)
    return dem


def library_kernels():
    """kernel_key of every __global__ entry of the built libdsmil_b200.so."""
    from dsmil_wsi_b200 import build
    dump, _ = _toolkit_tools()
    assert os.path.exists(build.LIB), "libdsmil_b200.so is not built"
    out = subprocess.run([dump, "-symbols", build.LIB], capture_output=True, text=True, check=True).stdout
    mangled = [line.split()[-1] for line in out.splitlines() if "STO_ENTRY" in line.split()]
    keys = [kernel_key(d) for d in demangle(mangled)]
    assert len(keys) == len(set(keys)), "two kernels share a key"
    return set(keys)


# ===================================================================================== CPU part: no device needed
def test_kernel_key_reads_both_demanglings():
    assert kernel_key("void dsmil::sm90::k_qmlp_sm90<(int)4, (int)512, (bool)1, (bool)0>(std::conditional<T4, "
                      "dsmil::sm90::QmlpModelsArgs, dsmil::sm90::QmlpArgs>::type)") == "k_qmlp_sm90<4,512,1,0>"
    assert kernel_key("void dsmil::sm90::k_qmlp_sm90<4, 512, true, false>(std::conditional<false, "
                      "dsmil::sm90::QmlpModelsArgs, dsmil::sm90::QmlpArgs>::type)") == "k_qmlp_sm90<4,512,1,0>"
    assert kernel_key("dsmil::k_argmax(const float *, long, int, unsigned long long *)") == "k_argmax"
    assert kernel_key("dsmil::k_argmax(float const*, long, int, unsigned long long*)") == "k_argmax"


def test_the_table_is_the_library():
    lib = library_kernels()
    missing = sorted(lib - set(KERNELS))
    stale = sorted(set(KERNELS) - lib)
    assert not missing and not stale, f"kernels without an entry: {missing}; entries without a kernel: {stale}"


def _case_index():
    idx = {}
    for prefix, mod in (("fwd", FW), ("bwd", BW)):
        for c in mod.ALL:
            idx[f"{prefix}:{c.name}"] = (prefix, c)
    return idx


def test_every_credit_names_a_case_and_every_exemption_a_test_file():
    idx = _case_index()
    here = os.path.dirname(os.path.abspath(__file__))
    for k, v in KERNELS.items():
        if isinstance(v, Exempt):
            assert os.path.exists(os.path.join(here, v.split(":")[0].split(" /")[0])), (k, v)
        else:
            assert v and all(c in idx for c in v), (k, v)


# ========================================================================================== GPU part (one H100)
def launched(fn):
    """kernel_key of every kernel of the library that fn() launches (torch.profiler, CUDA activities)."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    names = {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
    mangled = sorted(n for n in names if n.startswith("_Z"))
    plain = [n for n in names if not n.startswith("_Z")] + (demangle(mangled) if mangled else [])
    return {kernel_key(n) for n in plain if "dsmil::" in n}


def run_forward_case(case):
    lib = FW._lib_load()
    Xs = [b.X for b in FW.bags(case)]
    if case.route == "models":
        FW.run_models(case, lib, [FW._pack(FW.make_params(case, m)) for m in range(2)], Xs)
        return
    P = FW._pack(FW.make_params(case))
    if case.route == "single":
        FW.run_single(case, lib, P, Xs[0])
    elif case.route == "bags":
        FW.run_bags(case, lib, P, Xs)
    elif case.route == "value":
        FW.run_value(case, lib, P, Xs, FW.v_masks(case))
    else:
        for G in (1, 2, 3):
            for X in Xs:
                FW.run_shard_per_bag(case, P, X, G, crafted=G != 2)
            if case.tc_phase1 and min(case.Ns) >= G:
                FW.run_shard_bags(case, P, Xs, G)


SHARD_OPS = {"shard_bags": ("bag_ops", "bag_dev_ops"), "shard_per_bag": ("per_bag_ops",)}


def run_backward_case(case):
    if case.route == "single":
        BW.run_single(case, False)
    elif case.route == "bags":
        BW.run_bags(case, False)
    elif case.route == "dev":
        BW.run_dev(case, False)
    elif case.route == "models":
        for dev in (False, True):
            BW.run_models(case, False, dev)
    else:
        for ops in SHARD_OPS[case.route]:
            for G in (1, 2, 3):
                BW.run_shard(case, ops, G, False)


@pytest.mark.gpu
def test_every_case_launches_its_credited_kernels_and_together_they_launch_every_kernel():
    seen, by_case = set(), {}
    for cid, (kind, case) in _case_index().items():
        got = launched(lambda: (run_forward_case if kind == "fwd" else run_backward_case)(case))
        by_case[cid] = got
        seen |= got
    short = {cid: sorted(k for k, v in KERNELS.items() if not isinstance(v, Exempt) and cid in v and k not in got)
             for cid, got in by_case.items()}
    short = {cid: ks for cid, ks in short.items() if ks}
    assert not short, f"cases that did not launch kernels credited to them: {short}"
    never = sorted(k for k, v in KERNELS.items() if not isinstance(v, Exempt) and k not in seen)
    assert not never, f"kernels no conditioned case launched: {never}"
    unknown = sorted(seen - set(KERNELS))
    assert not unknown, f"launched kernels without an entry: {unknown}"
