"""CPU: the C-ABI library loads and exports every symbol include/xb200.h declares (no compute calls without a GPU)."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_symbols():
    src = open(os.path.join(ROOT, "include", "xb200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(xb_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    from xuance_b200 import _lib, build
    build.build()
    lib = ctypes.CDLL(_lib.LIB_PATH)
    names = _header_symbols()
    assert len(names) >= 20
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/xb200.h but not exported by libxb200.so"
    assert sorted(_lib.exported_symbols()) == names, "python binding table and header disagree"
    assert lib.xb_version() >= 100


def test_error_strings_and_argument_checks_without_gpu():
    from xuance_b200 import _lib
    lib = _lib.load()
    assert b"aligned" in lib.xb_error_string(-2)
    # argument validation happens before any CUDA call: NULL pointers are rejected with XB_EINVAL
    assert lib.xb_gae_scan(None, None, None, None, None, None, None, None, 4, 4, 0.99, 0.95, 1, None) == -1
    assert lib.xb_rollout_store(None, None, 16, None, None, 0, 0, 4, 0, None) == -1
    assert lib.xb_per_insert(None, None, None, 1, 3, 0, 0.5, None) == -1


def test_product_refuses_cpu():
    """No CPU fallback: buffers / learners raise on a non-CUDA device instead of silently running elsewhere."""
    import numpy as np
    import pytest
    from xuance_b200.common import DummyOnPolicyBuffer, Box, Discrete
    with pytest.raises(RuntimeError, match="CUDA"):
        DummyOnPolicyBuffer(Box(-1, 1, (3,), np.float32), Discrete(2), None, 2, 4, device="cpu")


def test_product_does_not_import_oracle():
    """oracle/ is test infrastructure: nothing under xuance_b200/ may import it."""
    bad = []
    for dp, _, fs in os.walk(os.path.join(ROOT, "xuance_b200")):
        for f in fs:
            if f.endswith(".py"):
                txt = open(os.path.join(dp, f)).read()
                if re.search(r"^\s*(from|import)\s+oracle\b", txt, flags=re.M):
                    bad.append(os.path.join(dp, f))
    assert not bad, bad


def test_every_entry_point_validates_before_touching_the_device():
    """Error behaviour of the C-ABI (include/xb200.h): bad sizes / NULL pointers / unsupported ranges are rejected with a
    negative XB_E* code before any CUDA call, so this runs without a GPU."""
    import ctypes
    from xuance_b200 import _lib
    lib = _lib.load()
    P = ctypes.c_void_p
    junk = P(0x1000)          # never dereferenced: validation fails first
    odd = P(0x1001)           # misaligned pointer
    EINVAL, EALIGN, ERANGE = -1, -2, -3
    assert lib.xb_rollout_store(junk, junk, 6, None, None, 0, 4, 8, 0, None) == EALIGN        # row_bytes % 4 != 0
    assert lib.xb_rollout_store(junk, junk, 16, None, None, 0, 4, 8, 8, None) == EINVAL       # t >= T
    assert lib.xb_rollout_store(junk, None, 16, None, None, 0, 4, 8, 0, None) == EINVAL       # dst without src
    assert lib.xb_gae_scan(junk, junk, junk, junk, junk, None, junk, junk, 0, 8, 0.99, 0.95, 1, None) == EINVAL
    assert lib.xb_gather_rows(junk, None, -1, 16, junk, None) == EINVAL
    assert lib.xb_gather_rows(junk, None, 4, 6, junk, None) == EALIGN
    assert lib.xb_gather_rows(junk, None, 0, 16, junk, None) == 0                              # empty batch is a no-op
    assert lib.xb_gather_obs(junk, None, 4, 84, 84, 3, junk, 2, None) == ERANGE                # NCHW needs C == 4
    assert lib.xb_gather_obs(junk, None, 4, 5, 5, 1, junk, 1, None) == EALIGN                  # H*W*C % 16 != 0
    assert lib.xb_gather_obs(junk, None, 4, 84, 84, 4, junk, 9, None) == EINVAL                # unknown format
    assert lib.xb_gather_scalars(junk, 10, None, 4, 2, junk, 5, junk, junk, None) == EINVAL    # adv_field >= F
    assert lib.xb_ppo_loss_fwd_bwd(junk, junk, junk, junk, junk, junk, 8, 65, 8, 0.2, 0.25, 0.01, 0, junk, junk, junk, junk, None) == ERANGE
    assert lib.xb_ppo_loss_fwd_bwd(junk, junk, junk, junk, junk, junk, 8, 4, 4, 0.2, 0.25, 0.01, 0, junk, junk, junk, junk, None) == EINVAL  # B_total < B
    assert lib.xb_ppo_loss_fwd_bwd(junk, junk, junk, None, junk, junk, 8, 4, 8, 0.2, 0.25, 0.01, 0, junk, junk, junk, junk, None) == EINVAL  # clip needs old_logp
    assert lib.xb_ppo_loss_fwd_bwd(junk, junk, junk, junk, junk, junk, 8, 4, 8, 0.2, 0.25, 0.01, 7, junk, junk, junk, junk, None) == EINVAL  # loss_kind
    assert lib.xb_ppo_loss_fwd_bwd(odd, junk, junk, junk, junk, junk, 8, 4, 8, 0.2, 0.25, 0.01, 0, junk, junk, junk, junk, None) == EALIGN
    assert lib.xb_per_insert(junk, junk, junk, 2, 16, 16, 0.5, None) == EINVAL                 # ptr >= cap
    assert lib.xb_per_sample(junk, junk, junk, 2, 12, 4, 2, 12, 1.0, junk, junk, junk, None) == EINVAL   # cap not 2^k
    assert lib.xb_per_sample(junk, junk, junk, 2, 16, 17, 2, 16, 1.0, junk, junk, junk, None) == EINVAL  # size > cap
    assert lib.xb_per_update(junk, junk, junk, junk, junk, 2, 16, 0, 0.5, None) == EINVAL
    assert lib.xb_dqn_td_fwd_bwd(junk, junk, None, junk, junk, junk, 0, 4, 0, 0.99, junk, junk, junk, junk, None) == EINVAL
    assert lib.xb_grad_sumsq(odd, 16, 1.0, junk, junk, None) == EALIGN
    assert lib.xb_adam_step(junk, junk, junk, junk, 16, junk, 0.9, 0.999, 1e-5, 0.5, None, 1.0, 0, None) == EINVAL  # clip without norm
    assert lib.xb_soft_update(junk, None, 16, 0.005, None) == EINVAL
    assert lib.xb_sac_actor_loss(junk, junk, junk, None, 8, 8, junk, junk, junk, junk, junk, None) == EINVAL
    assert lib.xb_qmix_mix_fwd(junk, junk, junk, junk, junk, 8, 17, 32, junk, None) == ERANGE   # n > 16
    assert lib.xb_qmix_select_fwd(junk, junk, junk, junk, junk, None, 0, 0, 5, 60, 12, 1, junk, junk, junk, junk, None) == EINVAL
    td = lambda rows_total: lib.xb_qmix_td(junk, junk, junk, junk, junk, junk, 4, 5, 6, 0.99, rows_total, junk, junk, junk, None)
    assert td(4 * 6 - 1) == EINVAL                     # rows_total is the global B*T: never below the local one
    assert td(0) == EINVAL
    four = (P * 4)(junk, junk, junk, junk)
    assert lib.xb_qmix_mix_fused_fwd(junk, junk, four, four, junk, junk, junk, junk, junk, junk, 128, 98, 5, 64, 32, junk, None) == ERANGE
    assert lib.xb_qmix_mix_fused_fwd(junk, junk, four, four, junk, junk, junk, junk, junk, junk, 128, 160, 5, 32, 32, junk, None) == ERANGE  # smem
    assert lib.xb_powf_libm(None, 0.5, junk, 4, None) == EINVAL
    # K10 / K11: rollout glue
    assert lib.xb_categorical_act(junk, junk, None, 8, 65, junk, None, junk, None, None) == ERANGE       # A > 64
    assert lib.xb_categorical_act(junk, junk, None, 8, 4, None, None, None, None, None) == EINVAL        # no output
    assert lib.xb_categorical_act(None, junk, None, 8, 4, junk, None, junk, None, None) == EINVAL
    assert lib.xb_rms_update_normalize(junk, 0, 4, junk, junk, 1e-4, 1, junk, 5.0, 1e-8, None) == EINVAL
    assert lib.xb_rms_update_normalize(junk, 8, 4, junk, junk, 1e-4, 0, None, 5.0, 1e-8, None) == EINVAL  # nothing to do
    # K12 (tensor-core layers) and its operand preparation
    taps = (ctypes.c_int8 * 64)()
    gg = lambda pa=2, pb=2, C=32, T=16, N=64, nt=64, ld=64, c0=0, w=junk, po=2: lib.xb_gemm_gather_tc(
        pa, pb, junk, 1024, w, 1024, None, None, 0, 0, 2, 21, 21, C, 10, 10, 2, 2, T, taps, taps, N, nt, 1, junk, 1024, po, None, 10,
        10, 1, 1, 0, 0, ld, c0, None, None)
    assert gg(pb=4) == EINVAL                          # at most 3 planes
    assert gg(pa=3, pb=2) == EINVAL                    # planes_a <= planes_b
    assert gg(po=4) == EINVAL                          # output planes
    assert gg(C=12) == ERANGE                          # channels per tap: multiple of 8 (one 16-byte unit)
    assert gg(T=65) == ERANGE                          # tap table
    assert gg(N=48, nt=48) == ERANGE                   # column tile % 32
    assert gg(N=96, nt=64, ld=96) == ERANGE            # N % n_tile
    assert gg(pa=3, pb=3, N=128, nt=128, ld=128) == ERANGE   # planes_b * n_tile <= 256 (one MMA spans the adjacent planes)
    assert gg(C=8, T=3) == ERANGE                      # K = T*C must be a multiple of the 64-deep stage
    assert gg(ld=32) == EINVAL                         # output row shorter than out_c0 + N
    assert gg(ld=68, c0=4) == EALIGN                   # 16-byte output segments
    assert gg(w=odd) == EALIGN
    # halo mode: argument validation that precedes any CUDA / driver call
    i16 = (ctypes.c_int16 * 16)()
    halo = lambda n_sub=1, n_chunks=9, W=10, hw=12, w0=-1, rows=24, B=2, hp=12, tabs=i16: lib.xb_gemm_halo_tc(
        3, 3, junk, 1024, W, rows, hw, w0, n_sub, n_chunks, tabs, tabs, junk, 1024, None, None, 0, 0, B, hp, 1, i16, i16, 64, 1,
        junk, 1024, 3, None, 10, 10, 1, 1, i16, i16, 64, 0, 0, None, None)
    assert halo(tabs=None) == EINVAL
    assert halo(n_sub=5) == ERANGE and halo(n_sub=2, n_chunks=9) == ERANGE      # at most 4 sub-items, 16 chunks in all
    assert halo(hw=8) == EINVAL                                                # the raster row must hold the tensor row
    assert halo(w0=1) == EINVAL and halo(rows=25) == EINVAL                     # pixel origin <= 0; in_rows = B * hp
    from xuance_b200._lib import XbPackJob
    jobs = (XbPackJob * 2)()
    for J in jobs:
        J.w, J.out, J.N, J.C, J.KH, J.KW, J.mode, J.n_taps, J.scale, J.planes = junk.value, junk.value, 8, 8, 3, 3, 0, 0, 1.0, 3
    pk = lambda n=2: lib.xb_pack_weights(ctypes.addressof(jobs), n, None)
    assert pk(0) == EINVAL and pk(17) == EINVAL
    jobs[1].planes = 4
    assert pk() == EINVAL
    jobs[1].planes, jobs[1].mode, jobs[1].n_taps = 3, 2, 17
    assert pk() == ERANGE                               # tap list
    jobs[1].n_taps = 2
    jobs[1].kh[1] = 3
    assert pk() == ERANGE                               # tap outside the kernel
    jobs[1].kh[1], jobs[1].w = 2, None
    assert pk() == EINVAL
    wg = lambda splits=1, out=junk, g_ld=64: lib.xb_wgrad_gather_tc(2, 2, junk, 1024, junk, 1024, g_ld, 1, 10, 10, 64, 10, 10, 1,
                                                                  1, 9, taps, taps, 64, 64, splits, out, None)
    assert wg(splits=5) == EINVAL                      # 100 sites cannot feed 5 splits
    assert wg(out=None) == EINVAL
    assert wg(g_ld=32) == EINVAL                       # gradient rows shorter than N
    assert lib.xb_wgrad_reduce(junk, 0, 64, 64, 3, 3, 1.0, junk, 0, None) == EINVAL
    assert lib.xb_split_bf16(junk, 64, 4, junk, None) == EINVAL
    assert lib.xb_split_bf16(odd, 64, 2, junk, None) == EALIGN
    assert lib.xb_pack_conv_weight(junk, 32, 4, 8, 8, 0, 1.0, junk, None) == EINVAL
    assert lib.xb_gather_obs_planes(junk, None, 4, 100, 2, junk, None) == EALIGN                        # row_bytes % 16
    assert lib.xb_gather_obs_planes(junk, None, 4, 28224, 5, junk, None) == EINVAL
    assert lib.xb_gather_obs_planes(junk, None, 0, 28224, 2, junk, None) == 0                           # empty batch
    for code in (EINVAL, EALIGN, ERANGE):
        assert lib.xb_error_string(code).startswith(b"xb200:")
