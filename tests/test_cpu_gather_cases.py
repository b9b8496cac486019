"""not-gpu: the batches of tests/test_gpu_gather.py reach every copy path of gather_pages_kernel.  From the plan's
offsets and each view's storage offset and strides, every row's path, byte head and byte tail are known without a GPU
(tests/gather_cases.py); if the cases are edited, this fails when they stop covering a path."""
from gather_cases import CASES, MAX_BATCH, NET, case_paths, is_fast, plan, row_path, shapes

FAST = ["w16", "w4", "shift1", "shift2", "shift3"]


def test_gather_cases_cover_every_path():
    have = set().union(*(case_paths(c) for c in CASES))
    for kind, ch in (("page", 3), ("mask", 1)):
        want = {(kind, (p, head, tail)) for p in FAST for head in (False, True) for tail in (False, True)}
        want |= {(kind, "short"), (kind, "generic%d" % ch)}
        assert want <= have, "uncovered %s paths: %s" % (kind, sorted(want - have, key=str))


def test_gather_cases_batch_structure():
    names = [c.name for c in CASES]
    assert len(set(names)) == len(names)
    assert all(1 <= len(c.pages) <= MAX_BATCH for c in CASES)
    assert any(len(c.pages) == MAX_BATCH for c in CASES) and any(len(c.pages) < MAX_BATCH for c in CASES)
    for c in CASES:
        assert c.masks is None if c.job == "pages" else shapes(c.masks) == shapes(c.pages), c.name
        entries, page_bytes, mask_bytes = plan(c)   # the planner takes every batch
        assert all(int(e["page_off"]) % 768 == 0 and int(e["mask_off"]) % 256 == 0 for e in entries)
        for img in c.pages + (c.masks or []):
            if img.view is not None:
                assert img.view.size[:2] == (img.h, img.w)
    # a one-row and a one-column device page between taller ones, and a 7016 x 4960 page at an odd byte offset
    for c in CASES:
        sh = shapes(c.pages)
        if any(sh[i][0] == 1 and sh[i - 1][0] > 1 and sh[i + 1][0] > 1 for i in range(1, len(sh) - 1)) and \
                any(sh[i][1] == 1 and sh[i - 1][0] > 1 and sh[i + 1][0] > 1 for i in range(1, len(sh) - 1)):
            break
    else:
        raise AssertionError("no batch puts one-row and one-column pages between tall ones")
    assert any(i.h == 7016 and i.w == 4960 and i.view is not None and i.view.offset % 2 == 1
               for c in CASES for i in c.pages)
    # host and device images in every run pattern: a host run first, in the middle, last, and all host
    patterns = {"".join("D" if i.view is not None else "H" for i in imgs)
                for c in CASES for imgs in (c.pages, c.masks or [])}
    assert any(p.startswith("H") and "D" in p for p in patterns)
    assert any(p.startswith("D") and p.endswith("D") and "H" in p for p in patterns)
    assert any(p.endswith("H") and "D" in p for p in patterns)
    assert any(set(p) == {"H"} for p in patterns if p)
    # both jobs, and pages the letterbox accepts at the net size in every ctd_submit_pages batch
    assert {c.job for c in CASES} == {"pages", "refine"} and NET % 64 == 0


def test_row_path_model():
    # the copy_same_phase / copy_shifted arithmetic at a few hand-checked rows
    assert row_path(0, 0, 48) == ("w16", 0, 3, 0)
    assert row_path(5, 5, 21) == ("w16", 11, 0, 10)
    assert row_path(5, 5, 40) == ("w16", 11, 1, 13)
    assert row_path(4, 8, 21) == ("w4", 0, 5, 1)
    assert row_path(1, 2, 21) == ("shift3", 2, 4, 3)       # d + 2 is aligned, s + 2 = 3 mod 4
    assert row_path(3, 0, 8) == ("shift3", 0, 2, 0)
    assert row_path(0, 3, 3) == ("shift1", 1, 0, 2)


def test_fast_flag_model():
    # the submit calls' fast rule: pages with sc == 1 and sw == 3, masks with sw == 1
    from gather_cases import _generic_masks, _generic_pages, window
    assert is_fast(window(2, 5, 3, 1, 16), 3) and is_fast(window(2, 5, 1, 1, 6), 1)
    assert [is_fast(i, 3) for i in _generic_pages()] == [False, False, False, True, False, False]
    assert [is_fast(i, 1) for i in _generic_masks()] == [False, False, False, False, True, False]
