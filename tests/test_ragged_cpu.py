"""CPU checks of the host-side tables of a ragged batch (every image its own label set): the union of the labels, the
packed text rows and the per-image offsets (lseg_net.ragged_label_table), and which label-set forms count as ragged."""
import pytest


def _mod():
    import lseg_b200  # noqa: F401
    from lseg_b200 import lseg_net
    return lseg_net


def test_table_disjoint_sets():
    m = _mod()
    union, rows, k, koff = m.ragged_label_table([["cat"], ["dog", "tree"], ["sky", "road", "car"]])
    assert union == ["cat", "dog", "tree", "sky", "road", "car"]
    assert rows == [0, 1, 2, 3, 4, 5]
    assert k == [1, 2, 3] and koff == [0, 1, 3]


def test_table_shared_labels_are_encoded_once():
    m = _mod()
    sets = [["cat", "other"], ["other", "dog", "cat"], ["cat", "other"]]
    union, rows, k, koff = m.ragged_label_table(sets)
    assert union == ["cat", "other", "dog"]
    assert k == [2, 3, 2] and koff == [0, 2, 5]
    # every image's packed rows name its own labels, in its own order
    for labels, o, n in zip(sets, koff, k):
        assert [union[r] for r in rows[o:o + n]] == labels
    assert len(rows) == sum(k) == koff[-1] + k[-1]


def test_table_repeated_label_within_an_image():
    m = _mod()
    union, rows, k, koff = m.ragged_label_table([["a", "a", "b"]])
    assert union == ["a", "b"] and rows == [0, 0, 1] and k == [3] and koff == [0]


@pytest.mark.parametrize("bad", [[[]], [["a"], "b"], [["a"], [3]], [("a",), None]])
def test_table_rejects_malformed_sets(bad):
    m = _mod()
    with pytest.raises(ValueError, match="labelsets"):
        m.ragged_label_table(bad)


def test_is_ragged():
    m = _mod()
    assert m.is_ragged([["a"], ["b", "c"]]) and m.is_ragged((["a"],)) and m.is_ragged([["a"], "b"])
    assert not m.is_ragged(["a", "b"]) and not m.is_ragged("") and not m.is_ragged("cat") and not m.is_ragged([])
