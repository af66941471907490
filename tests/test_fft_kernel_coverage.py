"""Every FFT-engine kernel of libsrtb_b200.so is accounted for: launched by a named case of test_gpu_fft_plans.py
(which checks, under torch.profiler, that the case did launch it) or listed with the reason no case can reach it.

The kernels are read from the built library with cuobjdump -elf and cu++filt. A kernel is named by its base name
and its integer template arguments (namespace, casts and type arguments dropped, true/false written 1/0), e.g.
fft_pass_kernel<7,16,1,1> for fft_pass_kernel<7, 16, MODE_COL, true, col_io<7, 16, true>>. The test fails when the
library has an FFT-engine kernel the table lacks, or the table names one the library lacks.
"""
import re
import shutil
import subprocess

import pytest

FFT_ENGINE = re.compile(r"^(fft_\w+|tiny_fft_kernel|r2c_post_kernel|r2c_col0_fixup_kernel)(<|$)")


def normalise(name: str) -> str:
    """base name + integer template arguments of a demangled kernel name (cu++filt or torch.profiler spelling)"""
    name = name.strip()
    if name.startswith("void "):
        name = name[5:]
    depth, base_end, args, cur = 0, None, [], ""
    for i, ch in enumerate(name):
        if ch == "<":
            if depth == 0 and base_end is None:
                base_end = i
            else:
                cur += ch
            depth += 1
        elif ch == ">":
            depth -= 1
            if depth == 0:
                args.append(cur)
                break
            cur += ch
        elif ch == "," and depth == 1:
            args.append(cur)
            cur = ""
        elif ch == "(" and depth == 0:
            base_end = i
            break
        elif depth >= 1:
            cur += ch
    base = name[:base_end].split("::")[-1].strip()
    if not args:
        return base
    ints = []
    for a in args:
        a = re.sub(r"\((?:int|bool|unsigned int|unsigned)\)", "", a).strip()
        a = {"true": "1", "false": "0"}.get(a, a)
        if re.fullmatch(r"-?\d+[uUlL]*", a):
            ints.append(str(int(a.rstrip("uUlL"))))
    return f"{base}<{','.join(ints)}>"


_TMA_REFUSED = "unreached: plain-load fallback taken only when the driver refuses a tensor map"

# kernel -> the test_gpu_fft_plans case that launches it, or "unreached: <reason>"
KERNEL_CASES = {
    'fft_bigrow_kernel<13,0,0,0>': 'test_c2c_vs_float64[k13-b5-off0-bwd]',
    'fft_bigrow_kernel<13,0,1,1>': 'test_block_route[bigrow_v1_8192]',
    'fft_bigrow_kernel<13,0,1,2>': 'test_block_route[bigrow_exact_8192]',
    'fft_bigrow_kernel<13,0,1,3>': 'test_block_route[sweep_bigrow_v3_8192]',
    'fft_bigrow_kernel<13,0,1,4>': 'test_block_route[bigrow_v4_8192_inverted]',
    'fft_bigrow_kernel<13,0,1,5>': 'test_block_route[bigrow_exact_8192]',
    'fft_bigrow_kernel<13,1,0,0>': 'test_c2c_vs_float64[k13-b5-off0-fwd]',
    'fft_bigrow_kernel<14,0,0,0>': 'test_c2c_vs_float64[k14-b3-off0-bwd]',
    'fft_bigrow_kernel<14,0,1,1>': 'test_block_route[sweep_bigrow_v1_16384]',
    'fft_bigrow_kernel<14,0,1,2>': 'test_block_route[sweep_bigrow_v2_16384]',
    'fft_bigrow_kernel<14,0,1,3>': 'test_block_route[bigrow_v3_16384]',
    'fft_bigrow_kernel<14,0,1,4>': 'test_block_route[sweep_bigrow_v4_16384]',
    'fft_bigrow_kernel<14,0,1,5>': 'test_block_route[bigrow_v3_16384]',
    'fft_bigrow_kernel<14,1,0,0>': 'test_c2c_vs_float64[k14-b3-off0-fwd]',
    'fft_col16_tma_kernel<7,16,0,0,0>': 'test_c2c_vs_float64[k21-b1-off0-bwd]',
    'fft_col16_tma_kernel<7,16,1,0,0>': 'test_c2c_vs_float64[k21-b1-off0-fwd]',
    'fft_col16_tma_kernel<7,16,1,1,0>': 'test_block_raw_format[NAOCPSR_SNAP1--8-22]',
    'fft_col16_tma_kernel<7,16,1,2,0>': 'test_block_raw_format[SIMPLE-8-22]',
    'fft_col16_tma_kernel<7,16,1,3,0>': 'test_block_raw_format[SIMPLE-4-22]',
    'fft_col16_tma_kernel<7,32,0,0,0>': 'test_c2c_vs_float64[k27-b1-off0-bwd]',
    'fft_col16_tma_kernel<7,32,1,0,0>': 'test_c2c_vs_float64[k27-b1-off0-fwd]',
    'fft_col16_tma_kernel<7,32,1,1,0>': 'test_block_raw_format[NAOCPSR_SNAP1--8-28]',
    'fft_col16_tma_kernel<7,32,1,2,0>': 'test_block_raw_format[SIMPLE-8-28]',
    'fft_col16_tma_kernel<7,32,1,3,0>': 'test_block_raw_format[SIMPLE-2-28]',
    'fft_col16_tma_kernel<8,16,0,0,0>': 'test_c2c_vs_float64[k15-b5-off0-bwd]',
    'fft_col16_tma_kernel<8,16,0,0,1>': 'test_block_route[long_n2_32768]',
    'fft_col16_tma_kernel<8,16,1,0,0>': 'test_c2c_vs_float64[k15-b5-off0-fwd]',
    'fft_col16_tma_kernel<8,16,1,1,0>': 'test_block_route[bigrow_v1_8192]',
    'fft_col16_tma_kernel<8,16,1,2,0>': 'test_block_raw_format[SIMPLE-8-23]',
    'fft_col16_tma_kernel<8,16,1,3,0>': 'test_block_raw_format[SIMPLE-4-23]',
    'fft_col16_tma_kernel<9,8,0,0,0>': 'test_c2c_vs_float64[k17-b5-off0-bwd]',
    'fft_col16_tma_kernel<9,8,0,0,1>': 'test_block_route[long_n0_131072_inverted]',
    'fft_col16_tma_kernel<9,8,1,0,0>': 'test_c2c_vs_float64[k17-b5-off0-fwd]',
    'fft_col16_tma_kernel<9,8,1,1,0>': 'test_block_raw_format[NAOCPSR_SNAP1--8-26]',
    'fft_col16_tma_kernel<9,8,1,2,0>': 'test_block_raw_format[SIMPLE-8-26]',
    'fft_col_tma_kernel<10,8,0>': 'test_c2c_vs_float64[k19-b5-off0-bwd]',
    'fft_col_tma_kernel<10,8,1>': 'test_c2c_vs_float64[k19-b5-off0-fwd]',
    'fft_col_tma_kernel<6,16,0>': 'test_c2c_vs_float64[k27-b1-off0-bwd]',
    'fft_col_tma_kernel<6,16,1>': 'test_c2c_vs_float64[k27-b1-off0-fwd]',
    'fft_pass_kernel<10,2,0,0>': 'test_c2c_vs_float64[k10-b3-off8-bwd]',
    'fft_pass_kernel<10,2,0,1>': 'test_c2c_vs_float64[k10-b3-off8-fwd]',
    'fft_pass_kernel<10,8,1,0>': 'test_c2c_vs_float64[k19-b5-off8-bwd]',
    'fft_pass_kernel<10,8,1,1>': 'test_c2c_vs_float64[k19-b5-off8-fwd]',
    'fft_pass_kernel<10,8,2,0>': _TMA_REFUSED,
    'fft_pass_kernel<10,8,2,1>': _TMA_REFUSED,
    'fft_pass_kernel<11,1,0,0>': 'test_c2c_vs_float64[k11-b5-off8-bwd]',
    'fft_pass_kernel<11,1,0,1>': 'test_c2c_vs_float64[k11-b5-off8-fwd]',
    'fft_pass_kernel<12,1,0,0>': 'test_c2c_vs_float64[k12-b3-off8-bwd]',
    'fft_pass_kernel<12,1,0,1>': 'test_c2c_vs_float64[k12-b3-off8-fwd]',
    'fft_pass_kernel<3,256,0,0>': 'test_c2c_vs_float64[k3-b5-off8-bwd]',
    'fft_pass_kernel<3,256,0,1>': 'test_c2c_vs_float64[k3-b5-off8-fwd]',
    'fft_pass_kernel<4,128,0,0>': 'test_c2c_vs_float64[k4-b3-off8-bwd]',
    'fft_pass_kernel<4,128,0,1>': 'test_c2c_vs_float64[k4-b3-off8-fwd]',
    'fft_pass_kernel<5,64,0,0>': 'test_c2c_vs_float64[k5-b5-off8-bwd]',
    'fft_pass_kernel<5,64,0,1>': 'test_c2c_vs_float64[k5-b5-off8-fwd]',
    'fft_pass_kernel<6,16,1,0>': _TMA_REFUSED,
    'fft_pass_kernel<6,16,1,1>': _TMA_REFUSED,
    'fft_pass_kernel<6,16,2,0>': _TMA_REFUSED,
    'fft_pass_kernel<6,16,2,1>': _TMA_REFUSED,
    'fft_pass_kernel<6,32,0,0>': 'test_c2c_vs_float64[k6-b3-off8-bwd]',
    'fft_pass_kernel<6,32,0,1>': 'test_c2c_vs_float64[k6-b3-off8-fwd]',
    'fft_pass_kernel<7,16,0,0>': 'test_c2c_vs_float64[k7-b5-off8-bwd]',
    'fft_pass_kernel<7,16,0,1>': 'test_c2c_vs_float64[k7-b5-off8-fwd]',
    'fft_pass_kernel<7,16,1,0>': 'test_c2c_vs_float64[k13-b5-off8-bwd]',
    'fft_pass_kernel<7,16,1,1>': 'test_c2c_vs_float64[k13-b5-off8-fwd]',
    'fft_pass_kernel<7,16,2,0>': _TMA_REFUSED,
    'fft_pass_kernel<7,16,2,1>': _TMA_REFUSED,
    'fft_pass_kernel<8,16,1,0>': 'test_c2c_vs_float64[k15-b5-off8-bwd]',
    'fft_pass_kernel<8,16,1,1>': 'test_c2c_vs_float64[k15-b5-off8-fwd]',
    'fft_pass_kernel<8,16,2,0>': _TMA_REFUSED,
    'fft_pass_kernel<8,16,2,1>': _TMA_REFUSED,
    'fft_pass_kernel<8,8,0,0>': 'test_c2c_vs_float64[k8-b3-off8-bwd]',
    'fft_pass_kernel<8,8,0,1>': 'test_c2c_vs_float64[k8-b3-off8-fwd]',
    'fft_pass_kernel<9,4,0,0>': 'test_c2c_vs_float64[k9-b5-off8-bwd]',
    'fft_pass_kernel<9,4,0,1>': 'test_c2c_vs_float64[k9-b5-off8-fwd]',
    'fft_pass_kernel<9,8,1,0>': 'test_c2c_vs_float64[k17-b5-off8-bwd]',
    'fft_pass_kernel<9,8,1,1>': 'test_c2c_vs_float64[k17-b5-off8-fwd]',
    'fft_pass_kernel<9,8,2,0>': _TMA_REFUSED,
    'fft_pass_kernel<9,8,2,1>': _TMA_REFUSED,
    'fft_row16_tma_kernel<10,4,0,0,0>': 'test_c2c_vs_float64[k10-b3-off0-bwd]',
    'fft_row16_tma_kernel<10,4,0,1,1>': 'test_block_route[row16_1024]',
    'fft_row16_tma_kernel<10,4,1,0,0>': 'test_c2c_vs_float64[k10-b3-off0-fwd]',
    'fft_row16_tma_kernel<11,2,0,0,0>': 'test_c2c_vs_float64[k11-b5-off0-bwd]',
    'fft_row16_tma_kernel<11,2,0,1,1>': 'test_block_route[row16_2048_inverted]',
    'fft_row16_tma_kernel<11,2,1,0,0>': 'test_c2c_vs_float64[k11-b5-off0-fwd]',
    'fft_row16_tma_kernel<12,1,0,0,0>': 'test_c2c_vs_float64[k12-b3-off0-bwd]',
    'fft_row16_tma_kernel<12,1,0,1,1>': 'test_block_route[row16_4096]',
    'fft_row16_tma_kernel<12,1,1,0,0>': 'test_c2c_vs_float64[k12-b3-off0-fwd]',
    'fft_row16_tma_kernel<8,16,0,0,0>': 'test_c2c_vs_float64[k8-b3-off0-bwd]',
    'fft_row16_tma_kernel<8,16,1,0,0>': 'test_c2c_vs_float64[k8-b3-off0-fwd]',
    'fft_row16_tma_kernel<9,8,0,0,0>': 'test_c2c_vs_float64[k9-b5-off0-bwd]',
    'fft_row16_tma_kernel<9,8,1,0,0>': 'test_c2c_vs_float64[k9-b5-off0-fwd]',
    'fft_row_tma_kernel<3,256,0,0>': 'test_c2c_vs_float64[k3-b5-off0-bwd]',
    'fft_row_tma_kernel<3,256,1,0>': 'test_c2c_vs_float64[k3-b5-off0-fwd]',
    'fft_row_tma_kernel<4,128,0,0>': 'test_c2c_vs_float64[k4-b3-off0-bwd]',
    'fft_row_tma_kernel<4,128,1,0>': 'test_c2c_vs_float64[k4-b3-off0-fwd]',
    'fft_row_tma_kernel<5,64,0,0>': 'test_c2c_vs_float64[k5-b5-off0-bwd]',
    'fft_row_tma_kernel<5,64,1,0>': 'test_c2c_vs_float64[k5-b5-off0-fwd]',
    'fft_row_tma_kernel<6,32,0,0>': 'test_c2c_vs_float64[k6-b3-off0-bwd]',
    'fft_row_tma_kernel<6,32,1,0>': 'test_c2c_vs_float64[k6-b3-off0-fwd]',
    'fft_row_tma_kernel<7,16,0,0>': 'test_c2c_vs_float64[k7-b5-off0-bwd]',
    'fft_row_tma_kernel<7,16,1,0>': 'test_c2c_vs_float64[k7-b5-off0-fwd]',
    'fft_row_tma_kernel<9,4,0,1>': 'test_block_route[unfused_512]',
    'fft_trans16_tma_kernel<7,16,0>': 'test_c2c_vs_float64[k14-b3-off8-bwd]',
    'fft_trans16_tma_kernel<7,16,1>': 'test_c2c_vs_float64[k14-b3-off8-fwd]',
    'fft_trans16_tma_kernel<8,16,0>': 'test_c2c_vs_float64[k16-b3-off0-bwd]',
    'fft_trans16_tma_kernel<8,16,1>': 'test_c2c_vs_float64[k16-b3-off0-fwd]',
    'fft_trans_r2c16_tma_kernel<7,8>': 'test_r2c_inplace_vs_float64[15-off0]',
    'fft_trans_r2c16_tma_kernel<8,8>': 'test_r2c_inplace_vs_float64[17-off0]',
    'fft_trans_r2c_tma_kernel<6,8>': 'test_r2c_inplace_vs_float64[14-off0]',
    'fft_trans_tma_kernel<10,8,0>': 'test_c2c_vs_float64[k20-b3-off0-bwd]',
    'fft_trans_tma_kernel<10,8,1>': 'test_c2c_vs_float64[k20-b3-off0-fwd]',
    'fft_trans_tma_kernel<6,16,0>': 'test_c2c_vs_float64[k13-b5-off8-bwd]',
    'fft_trans_tma_kernel<6,16,1>': 'test_c2c_vs_float64[k13-b5-off8-fwd]',
    'fft_trans_tma_kernel<9,8,0>': 'test_c2c_vs_float64[k18-b3-off0-bwd]',
    'fft_trans_tma_kernel<9,8,1>': 'test_c2c_vs_float64[k18-b3-off0-fwd]',
    'r2c_col0_fixup_kernel': 'test_r2c_inplace_vs_float64[14-off0]',
    'r2c_post_kernel<0>': 'test_r2c_inplace_vs_float64[1-off0]',
    'r2c_post_kernel<1>': 'test_r2c_inplace_vs_float64[19-off0]',
    'tiny_fft_kernel<0>': 'test_c2c_vs_float64[k1-b5-off0-bwd]',
    'tiny_fft_kernel<1>': 'test_c2c_vs_float64[k1-b5-off0-fwd]',
}


def library_kernels():
    import srtb_b200
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    cufilt = shutil.which("cu++filt") or "/usr/local/cuda/bin/cu++filt"
    try:
        r = subprocess.run([cuobjdump, "-elf", str(srtb_b200.LIB_PATH)], capture_output=True, text=True)
    except FileNotFoundError:
        pytest.skip("cuobjdump unavailable")
    if r.returncode != 0:
        pytest.skip("cuobjdump unavailable")
    syms = sorted(set(re.findall(r"\.text\.(\S+)", r.stdout)))
    dem = subprocess.run([cufilt], input="\n".join(syms), capture_output=True, text=True, check=True).stdout.split("\n")
    return {normalise(d) for d in dem if d.strip()}


def test_normalise_spellings():
    assert normalise("void srtb_b200::fft_pass_kernel<(int)7, (int)16, (int)1, (bool)1, "
                     "srtb_b200::col_io<(int)7, (int)16, (bool)1>>(T5, const float2 *)") == "fft_pass_kernel<7,16,1,1>"
    assert normalise("void srtb_b200::fft_pass_kernel<7, 16, 1, true, srtb_b200::col_io<7, 16, true> >"
                     "(srtb_b200::col_io<7, 16, true>, float2 const*)") == "fft_pass_kernel<7,16,1,1>"
    assert normalise("srtb_b200::r2c_col0_fixup_kernel(float2*, unsigned long)") == "r2c_col0_fixup_kernel"
    assert normalise("void tiny_fft_kernel<false>(float2*, int, unsigned long)") == "tiny_fft_kernel<0>"


def test_every_fft_kernel_is_in_the_table():
    lib = {k for k in library_kernels() if FFT_ENGINE.match(k)}
    assert lib, "no FFT-engine kernel found in the library"
    missing = sorted(lib - set(KERNEL_CASES))
    stale = sorted(set(KERNEL_CASES) - lib)
    assert not missing, f"kernels without a case or a reason: {missing}"
    assert not stale, f"table entries the library no longer has: {stale}"
    for k, case in KERNEL_CASES.items():
        assert case.startswith("unreached: ") or re.fullmatch(r"test_\w+(\[[\w.-]+\])?", case), (k, case)
