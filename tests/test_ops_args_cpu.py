"""CPU: every public tensor-taking op in `ops` states all of its tensor arguments through `ops._check` and rejects a
malformed call before any launch.  One row per op: a well-formed call on CPU tensors passes every device-free check and
fails only for not being on the GPU; every tensor argument reaches the device check; and each size relation the kernels
rely on is refused with a message that names the offending argument."""
import inspect
import re

import pytest
import torch

from naturalspeech2_pytorch_b200 import ops

B, N, D = 2, 8, 64
bf, i32, i64 = torch.bfloat16, torch.int32, torch.int64


def f(*s, dtype=torch.float32):
    return torch.zeros(*s, dtype=dtype)


def lens():
    return torch.ones(B, dtype=i32)


def _gemm():
    return dict(a=f(B, N, 64, dtype=bf), w=f(128, 64, dtype=bf), out=f(B, N, 128, dtype=bf), n=128,
                epilogue=ops.EPI_BF16, bias=f(128), film=f(B, 256))


def _gemm_f32():
    return dict(_gemm(), out=f(B, N, 128), epilogue=ops.EPI_F32, resid=f(B, N, 128))


def _rvq_ce():
    return dict(frames=f(6, 128), codebooks=f(2, 64, 128), cn2=f(2, 64), own_codes=f(6, 2, dtype=i64),
                target_codes=f(6, 2, dtype=i64))


def _attn_bwd():
    q = f(B, N, 64, dtype=bf)
    kv = f(B, 5, 64, dtype=bf)
    return dict(q=q, k=kv, v=kv.clone(), o=q.clone(), d_o=q.clone(), lse=f(B, 1, N), dq_accum=f(B, N, 64),
                dk=kv.clone(), dv=kv.clone(), heads=1)


def _rms_bwd():
    return dict(x=f(B, N, D), dh=f(B, N, D, dtype=bf), dxr=f(B, N, D), dxr_bf=f(B, N, D, dtype=bf), rows_per_batch=N,
                gamma=f(D), dgamma=f(D))


def _rms_bwd_film():
    return dict(_rms_bwd(), gamma=None, dgamma=None, film=f(B, 4 * D)[:, D:3 * D], dfilm=f(B, 2 * D))


def _wavenet():
    return dict(c=f(B, N, 2 * D, dtype=bf), dy=f(B, N, 2 * D, dtype=bf), dc=f(B, N, 2 * D, dtype=bf),
                film=f(B, 4 * D), dfilm=f(B, 4 * D), dim=D, groups=2, film_group_stride=2 * D)


def _rvq_encode():
    cb = f(2, 64, 128)
    return dict(frames=f(6, 128), codebooks=cb, prepared=(f(2 * 64 * 144, dtype=torch.float16), f(2, 64), f(2, 2)),
                codes=f(6, 2, dtype=i64), stats=f(8, dtype=i64))


# op -> (well-formed kwargs, {gap: (overriding kwargs, offending argument)}); several rows may test one op
CASES = {
    "gemm": (_gemm, {}),
    "gemm f32": (_gemm_f32, {}),
    "wgrad": (lambda: dict(dy=f(B, N, 128, dtype=bf), x=f(B, N, 64, dtype=bf), dw=f(128, 64), n=128, k=64), {}),
    "fold_conv_linear": (lambda: dict(w2=f(2, 4, 8), wc=f(2, 8, 6, 3), bc=f(2, 8), b2=f(2, 4), i_pad=8), {}),
    "dropout_": (lambda: dict(x=f(B, N, D), dropout=(1, 0, 0.5)), {}),
    "mask_rows": (lambda: dict(x=f(B, N, D), lens=lens()), {}),
    "pack_rows": (lambda: dict(a=f(B, 3, D, dtype=bf), a_lens=lens(), b=f(B, 4, D, dtype=bf), b_lens=lens(),
                               out=f(B, 7, D, dtype=bf)), {}),
    "attention": (lambda: dict(q=f(B, N, 128, dtype=bf), k=f(B, 5, 128, dtype=bf), v=f(B, 5, 128, dtype=bf),
                               out=f(B, N, 128, dtype=bf), heads=2, lse=f(B, 2, N), kv_lens=lens()), {
        "k batch": (dict(k=f(B + 1, 5, 128, dtype=bf)), "k"),
        "v length": (dict(v=f(B, 6, 128, dtype=bf)), "v"),
    }),
    "rmsnorm_film": (lambda: dict(x=f(B, N, D), out=f(B, N, D, dtype=bf), gamma=f(D), film=f(B, 3 * D)[:, D:]), {
        "gamma length": (dict(gamma=f(D - 1)), "gamma"),
        "film width": (dict(film=f(B, 2 * D - 1)), "film"),
    }),
    "rmsnorm_f32": (lambda: dict(x=f(B, N, D), out=f(B, N, D), gamma=f(D)), {}),
    "time_cond": (lambda: dict(times=f(B), freqs=f(8), w=f(32, 17), bias=f(32), out=f(B, 40)[:, 4:36]), {
        "w width": (dict(w=f(32, 16)), "w"),
        "bias length": (dict(bias=f(31)), "bias"),
        "freqs size": (dict(freqs=f(1, 8)), "freqs"),
    }),
    "small_linear": (lambda: dict(x=f(B, 20)[:, 2:18], w=f(32, 16), bias=f(32), out=f(B, 32), act=1), {
        "w against x": (dict(w=f(32, 15)), "w"),
        "bias length": (dict(bias=f(31)), "bias"),
    }),
    "cast_bf16": (lambda: dict(x=f(B, N, D), out=f(B * N, D, dtype=bf), add=f(B, N, D)), {}),
    "cond_inject": (lambda: dict(x=f(B, N, D), cproj=f(B, 5, D), out=f(B, N, D, dtype=bf),
                                 drop_mask=f(B, dtype=torch.bool), null_cond=f(D), cond_lens=lens()), {}),
    "select_rows": (lambda: dict(drop_mask=f(B, dtype=torch.bool), null_row=f(D), src=f(B, D),
                                 out=f(B, 3 * D)[:, D:2 * D]), {}),
    "select_rows bf16": (lambda: dict(drop_mask=f(B, dtype=torch.bool), null_row=f(4 * D), src=f(B, 4, D),
                                      out=f(B, 4, D, dtype=bf)), {}),
    "mean_rows": (lambda: dict(x=f(B, D, N).transpose(1, 2).contiguous()[:, :5], out=f(B, D), lens=lens()), {}),
    "transpose_cast": (lambda: dict(x=f(B, 2 * D, N)[:, :D], out=f(B, N, D, dtype=bf)), {}),
    "groupnorm_silu": (lambda: dict(x=f(B, N, D), weight=f(D), bias=f(D), groups=8, resid=f(B, N, D),
                                    out_f32=f(B, N, D), out_bf16=f(B, N, D, dtype=bf), lens=lens()), {
        "weight length": (dict(weight=f(D // 2)), "weight"),
        "bias length": (dict(bias=f(D // 2)), "bias"),
    }),
    "rowdot": (lambda: dict(x=f(B, N, D), w=f(1, D), bias=f(1), out=f(B, N)), {}),
    "expand_encodings": (lambda: dict(phon=f(B, 5, D), coarse=f(B, 5, dtype=i32), pitch_table=f(256, D),
                                      idx=f(B, N, dtype=i32)), {}),
    "embedding_bf16": (lambda: dict(ids=f(B, N, dtype=i64), table=f(10, D), out=f(B, N, D, dtype=bf), pad_id=0), {}),
    "q_sample": (lambda: dict(x0=f(B, N, D), noise=f(B, N, D), alpha=f(B), sigma=f(B), x_t=f(B, N, D),
                              target=f(B, N, D)), {}),
    "mse_rows": (lambda: dict(pred=f(B, N, D), target=f(B, N, D), out=f(B), scratch=f(B * 64), mean_out=f(())), {
        "out length": (dict(out=f(B + 1)), "out"),
        "scratch length": (dict(scratch=f(B * 64 - 1)), "scratch"),
    }),
    "ddim_step": (lambda: dict(x=f(B, N, D), v=f(B, N, D), alpha=f(B), sigma=f(B), alpha_next=f(B), sigma_next=f(B)), {}),
    "x_start_from_pred": (lambda: dict(x=f(B, N, D), pred=f(B, N, D), alpha=f(B), sigma=f(B), out=f(B, N, D)), {}),
    "cfg_combine": (lambda: dict(cond=f(B, N, D), null=f(B, N, D), scale=2.0, out=f(B, N, D)), {}),
    "rvq_prepare": (lambda: dict(codebooks=f(2, 64, 128)), {}),
    "rvq_encode": (_rvq_encode, {
        "frames width": (dict(frames=f(6, 64)), "frames"),
        "codes shape": (dict(codes=f(6, 3, dtype=i64)), "codes"),
    }),
    "rvq_decode": (lambda: dict(codes=f(6, 2, dtype=i64), codebooks=f(2, 64, 128), out=f(6, 128)), {}),
    "rvq_ce": (_rvq_ce, {}),
    "rvq_ce_bwd": (lambda: dict(_rvq_ce(), d_loss=f(1), row_scale=f(3), rows_per_sample=2, out=f(6, 256)), {}),
    "attention_bwd": (_attn_bwd, {
        "k batch": (dict(k=f(B + 1, 5, 64, dtype=bf)), "k"),
        "v length": (dict(v=f(B, 6, 64, dtype=bf)), "v"),
        "lse shape": (dict(lse=f(B, 1, N - 1)), "lse"),
    }),
    "rmsnorm_film_bwd": (_rms_bwd, {
        "dh size": (dict(dh=f(B, N - 1, D, dtype=bf)), "dh"),
        "dxr size": (dict(dxr=f(B, N, D - 4)), "dxr"),
        "gamma length": (dict(gamma=f(D + 1)), "gamma"),
        "dgamma length": (dict(dgamma=f(D - 1)), "dgamma"),
    }),
    "rmsnorm_film_bwd film": (_rms_bwd_film, {
        "film width": (dict(film=f(B, 2 * D - 1)), "film"),
        "film rows": (dict(film=f(B - 1, 2 * D)), "film"),
        "dfilm width": (dict(dfilm=f(B, D)), "dfilm"),
    }),
    "geglu_bwd": (lambda: dict(pre=f(B, N, 256, dtype=bf), dg=f(B, N, 128, dtype=bf)), {}),
    "wavenet_gate_bwd": (_wavenet, {
        "dy against c": (dict(dy=f(B, N + 1, 2 * D, dtype=bf)), "dy"),
        "dc against c": (dict(dc=f(B + 1, N, 2 * D, dtype=bf)), "dc"),
        "c columns": (dict(c=f(B, N, 2 * D - 1, dtype=bf)), "c"),
        "film columns": (dict(film=f(B, 4 * D - 1)), "film"),
    }),
    "colsum": (lambda: dict(t=f(B, N, 2 * D, dtype=bf)[:, :, :D], out=f(D)), {
        "out length": (dict(out=f(D - 1)), "out"),
    }),
    "group_sum": (lambda: dict(t=f(B, N, 2 * D, dtype=bf), out=f(B, N, D, dtype=bf), dim=D, groups=2), {
        "t against groups * out": (dict(t=f(B, N, D, dtype=bf)), "t"),
    }),
    "mse_bwd": (lambda: dict(pred=f(B, N, D), target=f(B, N, D), coef=f(B), out_bf=f(B, N, D, dtype=bf),
                             out_f32=f(B, N, D)), {}),
    "film_wgrad": (lambda: dict(dfilm=f(B, 3 * D)[:, D:2 * D], t=f(B, 32), dw=f(D, 32)), {}),
    "accum_bf16": (lambda: dict(acc=f(B, N, D), t=f(B, N, D, dtype=bf), acc_bf=f(B, N, D, dtype=bf)), {
        "acc_bf size": (dict(acc_bf=f(B, N, D - 1, dtype=bf)), "acc_bf"),
    }),
    "silu_bwd": (lambda: dict(pre=f(B, N, D, dtype=bf), dout=f(B, N, D, dtype=bf), dpre=f(B, N, D, dtype=bf)), {}),
    "embedding_bwd": (lambda: dict(ids=f(B, N, dtype=i64), de=f(B, N, D), dtable=f(10, D), pad_id=0), {}),
    "groupnorm_silu_bwd": (lambda: dict(x=f(B, N, D), weight=f(D), bias=f(D), groups=8, dy=f(B, N, D),
                                        dx=f(B, N, D, dtype=bf)), {}),
    "rowdot_bwd": (lambda: dict(x=f(B, N, D), w=f(D), pred=f(B, N), dpred=f(B, N), dx=f(B, N, D)), {}),
    "expand_encodings_bwd": (lambda: dict(dcond=f(B, N, 2 * D)[:, :, :D], coarse=f(B, 5, dtype=i32),
                                          idx=f(B, N, dtype=i32), dphon=f(B, 5, D), dtable=f(256, D)), {}),
    "add_rows_bcast": (lambda: dict(x=f(B, N, D), v=f(B, D), scale=0.5), {}),
    "maximum_path": (lambda: dict(value=f(B, 5, N), mask=f(B, 5, N)), {}),
    "lstm_seq": (lambda: dict(xproj=f(B, N + 2, 2048)[:, 2:], w_hh=f(2048, 512, dtype=bf), skip=f(B, N, 512),
                              out=f(B, N, 1024)[:, :, :512], out_bf16=f(B, N, 512, dtype=bf)), {}),
    "elu_pad": (lambda: dict(x=f(B, N, 32), out=f(B, N + 3, 64, dtype=bf), pad=3, raw=True), {}),
    "seanet_tail": (lambda: dict(x=f(B, N + 1, 32)[:, 1:], params=f(ops._lib.NS2_SEANET_TAIL_PARAMS), out=f(B, N)), {}),
    "seanet_head": (lambda: dict(x=f(B, 100), params=f(ops._lib.NS2_SEANET_HEAD_PARAMS), out=f(B, 102, 32, dtype=bf)),
                    {}),
}

# public functions of `ops` that take no tensor for a kernel: shape helpers, the launch counter and host-side lengths
NOT_TENSOR_OPS = {"set_sm_limit", "launch_count", "conv_segs", "conv3_segs", "conv_dgrad_segs", "lengths"}


def _op(case):
    return getattr(ops, case.split()[0])


@pytest.fixture(scope="module")
def lib():
    from naturalspeech2_pytorch_b200 import _lib, build
    build.build()
    return _lib.load()


def test_every_public_op_has_a_row():
    public = {name for name, fn in inspect.getmembers(ops, inspect.isfunction)
              if fn.__module__ == ops.__name__ and not name.startswith("_")}
    covered = {case.split()[0] for case in CASES}
    assert public - NOT_TENSOR_OPS - covered == set(), "ops without a row in CASES"
    assert covered <= public and NOT_TENSOR_OPS <= public


def _tensors(kwargs):
    for v in kwargs.values():
        for t in (v if isinstance(v, tuple) else (v,)):
            if isinstance(t, torch.Tensor):
                yield t


@pytest.mark.parametrize("case", CASES)
def test_well_formed_call_reaches_the_device_check(lib, case, monkeypatch):
    """Every device-free check accepts the call, it fails only for CPU tensors, and every tensor argument is among the
    ones `_check` puts through the device check."""
    kwargs = CASES[case][0]()
    seen = []
    check = ops._check

    def spy(*specs):
        seen.extend(id(s[1]) for s in specs if s[1] is not None)
        check(*specs)
    monkeypatch.setattr(ops, "_check", spy)
    before = lib.ns2_launch_count()
    with pytest.raises(ValueError, match="must be a CUDA tensor"):
        _op(case)(**kwargs)
    assert lib.ns2_launch_count() == before
    missed = [i for i, t in enumerate(_tensors(kwargs)) if id(t) not in seen]
    assert not missed, f"tensor arguments {missed} skip the device check"


GAPS = [(case, gap) for case, (_, gaps) in CASES.items() for gap in gaps]


@pytest.mark.parametrize("case, gap", GAPS)
def test_size_relation_is_refused(lib, case, gap):
    make, gaps = CASES[case]
    override, arg = gaps[gap]
    before = lib.ns2_launch_count()
    with pytest.raises(ValueError) as e:
        _op(case)(**{**make(), **override})
    assert re.match(rf"{arg}\b", str(e.value)) and "CUDA" not in str(e.value), str(e.value)
    assert lib.ns2_launch_count() == before
