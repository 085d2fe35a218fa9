"""The device assigns graph node ids by byte equality of memcmp-encoded keys (cozo_gpu_graph_stage_keys); that is only
the reference's BTreeMap<DataValue, u32> identity if byte equality of the encodings is DataValue equality."""
from tests.hostmod import load
from tests.test_graph_keys_gpu import mixed_keys


def test_encoding_equality_is_value_equality():
    h = load()
    keys = mixed_keys()
    keys += [list(k) if isinstance(k, list) else k for k in keys]      # equal values built twice
    enc = [h.memcmp_encode_value(k) for k in keys]
    for a, ea in zip(keys, enc):
        for b, eb in zip(keys, enc):
            assert (ea == eb) == (h.cmp(a, b) == 0), (a, b)
