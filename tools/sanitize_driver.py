"""Small-size pass over every shipped kernel, meant to run under compute-sanitizer (see tools/sanitize.sh)."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

from unionml_b200.engine import Engine  # noqa: E402

z = np.load("tests/golden/digits_lr.npz")
g = np.load("tests/golden/mlp_64_32_10.npz")
eng = Engine(0)
m = eng.load_linear(z["coef"], z["intercept"])
mlp = eng.load_mlp(g["w1"], g["b1"], g["w2"], g["b2"])
X = np.random.default_rng(0).integers(0, 17, size=(40_001, 64), dtype=np.uint8).astype(np.float32)
b = eng.stage(np.asfortranarray(X.astype(np.float64)))  # feature-major float64 source -> transpose kernel
for exact in (True, False):
    eng.predict(m, b, exact=exact)
    eng.predict_mlp(mlp, b, exact=exact)
eng.predict_host(m, X, exact=True, chunk_rows=4096)
buf = eng.device_alloc(b.n_rows)
eng.predict_peers(m, b, [buf.ptr], 0, exact=True, want_stats=True, label_bytes=1)
eng.take_labels(buf.ptr, b.n_rows, np.arange(10.0), label_bytes=1)
# round 2: tensor-core MLP kernel (+ peer stores), CUDA-core MLP kernel on float rows, re-score from
# the caller's float64 values, online small-batch kernel, predict_proba, MLP host pipeline, asynchronous host call
import os as _os

eng.predict_mlp_peers(mlp, b, [buf.ptr], 0, exact=True, want_stats=True, label_bytes=1)
Xf = np.random.default_rng(1).standard_normal((20_001, 64))
bf = eng.stage(Xf)
eng.predict_mlp(mlp, bf, exact=True)                     # general floats: FFMA kernel
eng.predict_host(m, Xf, exact=True, chunk_rows=4096)     # float64 source: re-score reads the raw chunk
eng.predict_host(m, np.asfortranarray(Xf[:32]), exact=True)   # online shape: zero-copy kernel, graph replay
eng.predict_host(m, np.asfortranarray(Xf[:32]), exact=True)
eng.predict_proba(m, b)
eng.predict_mlp_host(mlp, X.astype(np.float64), chunk_rows=4096)
eng.predict_host_list(m, X.astype(np.float64), [float(c) for c in range(10)], chunk_rows=4096, asynchronous=True)
m0 = eng.load_linear(np.zeros((5, 64)), np.zeros(5))    # every row a tie: the queue backs up, scoring warps re-score their own rows
eng.predict(m0, b, exact=True)
# fp64 re-score with the feature-major weight table: two rounds of classes (C = 20 -> generic all-rows kernel), an odd
# class count behind the tile kernel, and a wide model whose table is staged in shared memory (F = 784)
rng = np.random.default_rng(4)
m20 = eng.load_linear(rng.standard_normal((20, 64)), rng.standard_normal(20))
eng.predict(m20, b, exact=True)
m3 = eng.load_linear(rng.standard_normal((3, 64)), rng.standard_normal(3))
eng.predict(m3, bf, exact=True)
X784 = (rng.integers(0, 256, size=(6_001, 784)) / 255.0)
m784 = eng.load_linear(rng.standard_normal((10, 784)) * 0.05, rng.standard_normal(10))
eng.predict(m784, eng.stage(X784), exact=True)
eng.predict_host(m784, X784, exact=True, chunk_rows=2048)
# MLP online route (mlp_small_kernel): a feature-major float64 block (capture, then replay) and a 1-row int64 request
eng.predict_mlp_host(mlp, np.asfortranarray(Xf[:32]))
eng.predict_mlp_host(mlp, np.asfortranarray(Xf[:32]))
eng.predict_mlp_host(mlp, X[:1].astype(np.int64))
# MLP top-k: tensor-core and CUDA-core top-k forms with their fp64 re-score, the fp64 kernel for k > 5, device outputs
# 4 bytes off 16-byte alignment, indices only, and the hit count
for batch in (b, bf):
    for k in (1, 3, 5, 10):
        eng.predict_mlp_topk(mlp, batch, k, exact=True)
        eng.predict_mlp_topk(mlp, batch, k, exact=False, want_proba=False)
kb = eng.device_alloc(4 * (3 * b.n_rows + 1))
pb = eng.device_alloc(4 * (3 * b.n_rows + 1))
eng.predict_mlp_topk(mlp, b, 3, idx_device_ptr=kb.ptr + 4, proba_device_ptr=pb.ptr + 4)
eng.predict_mlp_topk(mlp, b, 3, want_proba=False, idx_device_ptr=kb.ptr)
eng.count_topk_hits(kb.ptr, 3, b.n_rows, np.arange(10.0), np.zeros(b.n_rows))
# compact fp16 rows: `b` holds integers, so staging packed its fp16 copy and the linear predicts above ran the tile
# kernel's fp16 schedule; here also pinned float32 rows (finite-scan staging), F = 7 (the box's first 32 features
# only) with peer stores at an odd offset, and the same batch on the fp32 route through the test hook
bp = eng.pinned_empty(X.shape, np.float32)
bp[:] = X
b16 = eng.stage(bp)
for exact in (True, False):
    assert eng.predict(m, b16, exact=exact)[1]["x_elem_bytes"] == 2
m7 = eng.load_linear(rng.standard_normal((10, 7)), rng.standard_normal(10))
b7 = eng.stage(X[:, :7])
eng.predict(m7, b7, exact=True)
buf7 = eng.device_alloc(b7.n_rows + 3)
eng.predict_peers(m7, b7, [buf7.ptr], 3, exact=True, want_stats=True, label_bytes=1)
_os.environ["UML_B200_COMPACT_ROWS"] = "0"
assert eng.predict(m, b16, exact=True)[1]["x_elem_bytes"] == 4
del _os.environ["UML_B200_COMPACT_ROWS"]
# 256-row items of the fp16 schedule with the ring at its 4-item floor: ragged last items (40_001 = 156 x 256 + 65 rows
# ends inside the item's first box, 155 x 256 + 200 inside its second), uint8 peer stores at an odd offset, and a
# 16-class model (8 rows of 17 accumulators per lane, 255 registers)
_os.environ["UML_B200_STAGES"] = "4"
m16 = eng.load_linear(rng.standard_normal((16, 64)), rng.standard_normal(16))
b200 = eng.stage(X[: 155 * 256 + 200])
buf16 = eng.device_alloc(b16.n_rows + 1)
for mm in (m, m16):
    for bb in (b16, b200):
        for exact in (True, False):
            assert eng.predict(mm, bb, exact=exact)[1]["x_elem_bytes"] == 2
        eng.predict_peers(mm, bb, [buf16.ptr], 1, exact=True, want_stats=True, label_bytes=1)
del _os.environ["UML_B200_STAGES"]
# byte rows: `b16` and `b200` hold integers 0..16, so staging also packed their byte copies and the EXACT predicts above
# took the tensor-core schedule on them; here that schedule (x_read_bytes 1) at its 3-item ring floor and at full
# depth, a ragged last item, 10 and 16 classes, uint8 peer stores at an odd offset, and the fp16 tensor-core schedule on
# the same batches (UML_B200_COMPACT_ROWS=2, x_read_bytes 2)
for stages in ("1", None):
    if stages:
        _os.environ["UML_B200_STAGES"] = stages
    for env, read in (("1", 1), ("2", 2)):
        _os.environ["UML_B200_COMPACT_ROWS"] = env
        for mm in (m, m16):
            for bb in (b16, b200):
                assert eng.predict(mm, bb, exact=True)[1]["x_read_bytes"] == read
                eng.predict_peers(mm, bb, [buf16.ptr], 1, exact=True, want_stats=True, label_bytes=1)
    del _os.environ["UML_B200_COMPACT_ROWS"]
    _os.environ.pop("UML_B200_STAGES", None)
# float64 probabilities (the scores kernel's softmax / sigmoid epilogue): binary, C = 10 (one class group, in the strip),
# C = 40 (grouped, normalised in global memory), F = 784 (W from global memory), host and resident, a device output
# 8 bytes off 16-byte alignment
mb = eng.load_linear(rng.standard_normal((1, 64)), rng.standard_normal(1))
m40 = eng.load_linear(rng.standard_normal((40, 64)), rng.standard_normal(40))
b64 = eng.stage(Xf[:3_001], keep_f64=True)
for mm in (mb, m, m40):
    for log in (False, True):
        eng.predict_proba_f64(mm, b64, log=log)
        eng.predict_proba_f64_host(mm, np.asfortranarray(Xf[:3_001]), log=log, chunk_rows=1024)
        eng.predict_proba_f64_host(mm, X[:4_001].astype(np.uint8), log=log)
for log in (False, True):
    eng.predict_proba_f64(m784, eng.stage(X784, keep_f64=True), log=log)
    eng.predict_proba_f64_host(m784, X784, log=log, chunk_rows=2048)
pf = eng.device_alloc(8 * (10 * b64.n_rows + 2))
eng.predict_proba_f64(m, b64, out_device_ptr=pf.ptr + 8, want_stats=True)
# MLP probabilities and top-k from host rows: the online kernel's two record forms (1 and 32 rows, capture then replay,
# k = 3 and k = C), and a mixed frame through the pipeline - integer rows first, so the tensor cores are picked and flag
# the later general-float rows for the flagged-row float64 probabilities and top-k
for rows in (1, 32):
    for _ in range(2):
        eng.predict_mlp_proba_host(mlp, Xf[:rows])
        eng.predict_mlp_topk_host(mlp, Xf[:rows], 3)
        eng.predict_mlp_topk_host(mlp, Xf[:rows], 10, exact=False)
mixed = np.concatenate([X[:4096].astype(np.float64), Xf[:3_001]])
eng.predict_mlp_proba_host(mlp, mixed, chunk_rows=2048)
for exact in (True, False):
    eng.predict_mlp_topk_host(mlp, mixed, 3, exact=exact, chunk_rows=2048)
print("sanitizer driver ok")
