"""The emulated copy of allreduce_nvls_kernel without a GPU (tests/nvls_emulate.py): it is the product kernel with its
two multimem statements replaced and nothing else, a kernel whose statements change fails loudly instead of testing
stale code, the copy compiles for sm_90a with no multicast instruction and no spills, the product kernel keeps both
multicast instructions (the reduction by its opcode, the store by its statement), and every named mutation applies at
exactly one place."""
import re

import pytest

import nvls_emulate as emu
from kernel_tools import kernel_sass

KERNEL_RE = r"^_ZN3cdp21allreduce_nvls_kernelE"
MULTICAST = re.compile(r"LDGMC|MULTIMEM")


@pytest.fixture(scope="module")
def built(tmp_path_factory):
    return emu.build(tmp_path_factory.mktemp("nvls_emulate"), ptxas_verbose=True)


def kernel_text():
    with open(emu.KERNEL) as f:
        return f.read()


def test_the_copy_replaces_the_two_multimem_statements_and_nothing_else():
    text = kernel_text()
    out = emu.generate(text)
    assert 'asm volatile("multimem' in text and 'asm volatile("multimem' not in out
    assert out.count(emu.LD_REDUCE_CALL) == 1 and out.count(emu.STORE_CALL) == 1
    # every other line is the product's, in order
    kept = [l for l in out.splitlines() if l.strip() not in (emu.LD_REDUCE_CALL, emu.STORE_CALL)]
    assert all(l in text.splitlines() for l in kept)
    assert len(text.splitlines()) - len(kept) == 4  # one line of ld_reduce, three of st


@pytest.mark.parametrize("edit", ["ld_twice", "st_twice", "ld_reworded", "st_reworded"])
def test_a_kernel_whose_statements_change_fails_to_generate(edit):
    text = kernel_text()
    ld, st = emu.LD_REDUCE.search(text).group(0), emu.STORE.search(text).group(0)
    changed = {"ld_twice": text.replace(ld, ld + "\n  " + ld),
               "st_twice": text.replace(st, st + "\n    " + st),
               "ld_reworded": text.replace(ld, ld.replace(".relaxed.sys", ".relaxed.gpu")),
               "st_reworded": text.replace(st, st.replace(".v4.f32", ".v2.f64"))}[edit]
    assert changed != text
    with pytest.raises(AssertionError):
        emu.generate(changed)


def test_an_edit_beside_the_statements_reaches_the_copy():
    """The copy is made from the file as it stands, so an edit elsewhere in the kernel is in the copy too."""
    text = kernel_text().replace("fw / (kUnitBytes / 8);", "fw / (kUnitBytes / 8);  // edited", 1)
    assert "// edited" in emu.generate(text)


@pytest.mark.parametrize("name", sorted(emu.MUTATIONS))
def test_every_mutation_applies_at_exactly_one_place(name):
    clean = emu.generate()
    mutated = emu.generate(mutation=name)
    old, new = emu.MUTATIONS[name]
    assert clean.count(old) == 1 and mutated.count(old) == 0 and mutated.count(new) == clean.count(new) + 1


def test_the_copy_compiles_for_sm_90a_with_no_multicast_instruction_and_no_spills(built):
    lib, ptxas = built
    _, sass = kernel_sass(lib, KERNEL_RE)
    assert not [t for t in sass if MULTICAST.search(t)]
    props = re.findall(r"Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads", ptxas)
    nvls = [p for p in props if "allreduce_nvls_kernelE" in p[0]]
    assert len(nvls) == 1 and nvls[0][2:] == ("0", "0"), props
    # the emulated reduction: one 8-byte system-scope load per member in a loop, the store a 16-byte one
    assert any(t.startswith("LDG.E.64.STRONG.SYS") for t in sass)


def test_the_host_harness_exports_its_entry_points(built):
    import ctypes as C

    lib = C.CDLL(built[0])
    for name in ("nvls_emul_open", "nvls_emul_call", "nvls_emul_corrupt", "nvls_emul_close", "nvls_emul_dims",
                 "nvls_emul_device", "nvls_emul_error"):
        assert hasattr(lib, name), name
    dims = (C.c_uint64 * 3)()
    lib.nvls_emul_dims(dims)
    assert list(dims) == [24, 65, 4 * 24 * 65 + 2 * 24 + 1]


def test_the_product_kernel_keeps_both_multicast_instructions(pkg):
    """The emulation replaces what the product kernel still issues.  Its SASS holds 32 multimem.ld_reduce (LDGMC) and
    the 16-byte system-scope stores multimem.st compiles to (STG.E.128.STRONG.SYS, the opcode of an ordinary store too,
    so the source pins the store statement itself); its source holds one statement of each."""
    _, sass = kernel_sass(pkg.abi.LIB_PATH, KERNEL_RE)
    assert len([t for t in sass if re.match(r"(@!?U?P\w+ )?LDGMC\.E\.ADD\.64\.STRONG\.SYS ", t)]) == 32
    assert len([t for t in sass if re.match(r"(@!?U?P\w+ )?STG\.E\.128\.STRONG\.SYS ", t)]) >= 16
    text = kernel_text()
    assert len(emu.LD_REDUCE.findall(text)) == 1 and len(emu.STORE.findall(text)) == 1
