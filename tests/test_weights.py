"""Weight tooling (SURVEY 8(f) rank 3): the direct checkpoint -> blob exporter must produce the bytes
of the reference pipeline (dump_rnnoise_weights.py --quantize -> C compiler -> dump_weights_blob)."""
import os
import sys

import numpy as np
import pytest

from oracle.make_models import REF
from rnnoise_b200 import weights

HERE = os.path.dirname(os.path.abspath(__file__))
MODELS = os.path.join(HERE, "golden", "models")


def _diff(a, b):
    """First differing record, for a readable failure."""
    ra, rb = weights.read_blob(a), weights.read_blob(b)
    assert [r[0] for r in ra] == [r[0] for r in rb]
    for (n, t, x), (_, t2, y) in zip(ra, rb):
        assert t == t2, n
        assert x.shape == y.shape, (n, x.shape, y.shape)
        assert np.array_equal(x.view(np.uint8), y.view(np.uint8)), (n, int(np.sum(x != y)))


def test_blob_roundtrip_is_byte_identical():
    for name in ("default", "little", "g256", "tiny"):
        raw = open(os.path.join(MODELS, name + ".bin"), "rb").read()
        assert weights.write_blob(weights.read_blob(raw)) == raw


def test_read_blob_rejects_malformed():
    raw = open(os.path.join(MODELS, "tiny.bin"), "rb").read()
    with pytest.raises(ValueError):
        weights.read_blob(raw[:-32])
    with pytest.raises(ValueError):
        weights.read_blob(b"XXXX" + raw[4:])
    bad = bytearray(raw); bad[16:20] = (1 << 30).to_bytes(4, "little")   # block_size past the end
    with pytest.raises(ValueError):
        weights.read_blob(bytes(bad))


def test_exporter_matches_reference_pipeline_on_committed_checkpoint(tmp_path):
    out = str(tmp_path / "tiny.bin")
    blob = weights.export_checkpoint(os.path.join(MODELS, "tiny_ckpt.npz"), out)
    ref = open(os.path.join(MODELS, "tiny.bin"), "rb").read()
    _diff(blob, ref)
    assert blob == ref and open(out, "rb").read() == ref
    assert weights.describe(blob)["cond"] == 96 and weights.describe(blob)["gru"] == 128


# needs the reference's Python model definition where oracle/make_models.py looks for it ($RNNOISE_REFERENCE); skipped
# where it is absent, because no reference source may be stored in this repository
@pytest.mark.skipif(not os.path.isdir(os.path.join(REF, "torch", "rnnoise")), reason="needs the reference model definition")
@pytest.mark.parametrize("name", ["default", "hot", "little", "g256", "little_b"])
def test_exporter_matches_reference_pipeline_on_seeded_models(name, tmp_path):
    """Rebuild the seeded checkpoint with the reference's model class (as oracle/make_models.py did)
    and export it directly: same bytes as the committed blob made through the C detour."""
    sys.path.insert(0, os.path.join(HERE, "..", "oracle"))
    import make_models
    ck = str(tmp_path / "ck.pth")
    make_models.make_ckpt(ck, **make_models.SPECS[name])
    blob = weights.export_checkpoint(ck, None)
    ref = open(os.path.join(MODELS, name + ".bin"), "rb").read()
    _diff(blob, ref)
    assert blob == ref


def test_exported_blob_loads_in_the_product_parser_and_port(tmp_path):
    """A blob written by the exporter is accepted by the C loader of the product (dims inferred from array
    sizes) and by the oracle port; a blob with a perturbed weight still parses (weights are data), one with a
    broken sparse index does not."""
    import ctypes as C
    import rnnoise_b200
    from oracle.portbind import Port
    out = str(tmp_path / "m.bin")
    blob = weights.export_checkpoint(os.path.join(MODELS, "tiny_ckpt.npz"), out)
    L = rnnoise_b200.lib()
    m = L.rnnoise_model_from_filename(out.encode())
    assert m
    L.rnnoise_model_free(m)
    assert Port(out).model
    recs = weights.read_blob(blob)
    idx = next(i for i, r in enumerate(recs) if r[0] == "gru1_input_weights_idx")
    broken = recs[idx][2].copy(); broken[0] += 1            # first block count no longer matches the weights
    recs[idx] = (recs[idx][0], recs[idx][1], broken)
    bad = weights.write_blob(recs)
    assert not L.rnnoise_model_from_buffer(bad, len(bad))


def test_sparse_index_overflow_and_repeated_positions_are_rejected():
    """ADVICE r1: a block count of INT_MAX must not overflow the parser's bounds check, and a position repeated
    inside one output block (which the reference's sparse kernel would ACCUMULATE, vec_avx.h:778-828, while a
    dense expansion overwrites) is refused instead of being mis-read."""
    import rnnoise_b200
    L = rnnoise_b200.lib()
    blob = open(os.path.join(MODELS, "tiny.bin"), "rb").read()
    assert L.rnnoise_model_from_buffer(blob, len(blob))
    for mutate in ("intmax", "repeat", "descending"):
        recs = weights.read_blob(blob)
        i = next(k for k, r in enumerate(recs) if r[0] == "gru2_recurrent_weights_idx")
        idx = recs[i][2].copy()
        assert idx[0] >= 2
        if mutate == "intmax":
            idx[0] = 2**31 - 1
        elif mutate == "repeat":
            idx[2] = idx[1]
        else:
            idx[1], idx[2] = idx[2], idx[1]
        recs[i] = (recs[i][0], recs[i][1], idx)
        bad = weights.write_blob(recs)
        assert not L.rnnoise_model_from_buffer(bad, len(bad)), mutate
