"""Hand-written and fuzzed corpora for the parity tests (test infrastructure)."""
import random

import numpy as np

EXT = {"other": 0, "py": 1, "cc": 2, "cpp": 3, "java": 4, "c": 5, "h": 6}

PY_SAMPLE = b'''import unittest
from mock import patch

class SkillTest(object):
    """Assert that the gui can set gui variables."""
    def setUp(self):
        self.x = 1
        assert self.x

class TestThing(unittest.TestCase):
    def test_docker_agent_init(monkeypatch, runner_token):
        agent = DockerAgent()
        assert agent
        assert agent.labels == []
        assert agent.name == "agent"
        assert not agent.no_pull
        assert "Schedule not found" in str(exc.value)
        assert result == 0, "Repo did not pass Black formatting!"
        assert x is not None
        assert res.mapped == True
        assert loss[-1] < loss[0] * data.convergence
        assert sys.version_info >= (3, 6)
        assert a <= b
        assert a != b
        assert a > b
        assert(x)
        assert
        assert\t
    def test_more(self):
        self.assertEqual(a, b)
        self.assertEqual (a, b)
        self.assertEquals(a, b)
        self.assert_(a)
        self.assertListEqual(a, b)
        self.assertWeirdCustomThing(a)
        mock.assert_called_once_with(1)
        service.list_player.set_media_list.assert_called_with(x)
        parser.add_argument('-f', '--filename', dest='filename', default="/tmp/test.wav")
        except AssertionError:
        response.getTransform(assert_me)
        # TODO assert Service is Available
    async def test_set_multiple(self):
        x = GPUAssert(y)
classifier = 3
class\tTabbed:
'''

CC_SAMPLE = b'''#include "gtest/gtest.h"
#include "modules/perception/fusion/common/dst_evidence.h"

namespace apollo {
class DSTEvidenceTest : public ::testing::Test {
 public:
  DSTEvidenceTest()
      : sensor1_dst_("test"), sensor2_dst_("test"), fused_dst_("test") {
    dst_manager->AddApp("test", fod_subsets, fod_subset_names);
    vec_equal_ = [](const std::vector<double> &vec,
                    const std::vector<double> &gt) {
      CHECK_EQ(vec.size(), gt.size());
      for (size_t i = 0; i < vec.size(); ++i) {
        EXPECT_NEAR(vec[i], gt[i], 1e-6);
      }
    };
  }
  ~DSTEvidenceTest() {}
  void assign_dst_test() {
    EXPECT_DOUBLE_EQ(dst_vec[i], dst_vec_gt[i]);
  }
};
TEST_F(DSTEvidenceTest, assign_test) {
  ASSERT_TRUE(sensor1_dst_.SetBbaVec(sensor1_data));
  EXPECT_EQ(latest_observed_msg_ptr->class_name(), "BlockerTest");
  EXPECT_STREQ("a", "b");
  EXPECT_CALL(mock, Foo());
  EXPECT_THROW(f(), std::exception);
  EXPECT_FLOAT_EQ(1.0f, x);
  else ASSERT_EQ(1, 2);
  // EXPECT_EQ(a, b);
  RAPIDJSON_ASSERT(x);
  FOR_EACH(assertion, list) {
  static_assert(sizeof(int) == 4, "int");
  EXPECT_GE(a, b); EXPECT_LE(a, b);
}
  TEST_F(Indented, fixture) {
TEST(TestSuite, CheckGenerateAnchors) {
  void CreateTestMapNode(unsigned int m, unsigned int n,
  EXPECT_LT(a,
            b);
}
'''

JAVA_SAMPLE = b'''package org.deepspeech.libdeepspeech.test;
public class MapDecodeTest {
    @Test public void testDoubleInitialize() throws Exception {
        assertEquals("org.deepspeech.libdeepspeech.test", appContext.getPackageName());
        assert (audioFormat == 1); // 1 is PCM
        assertTrue(x);
        Assert.assertEquals(1, 2);
        assertNull(y);
        assertThat(z, is(1));
    }
    public void mobilityOperationEncodeTest() {
        assertArrayEquals(a, b);
    }
}
'''

EDGE_FILES = [
    (b"", 1), (b"\n", 1), (b"\n\n\n", 2), (b"a", 1), (b"a\n", 1), (b"a\nb", 2), (b"\r\n\r\n", 1),
    (b"assert x\r\nEXPECT_EQ(a, b);\r\n", 2), (b"assert", 1), (b"x" * 5000, 1),
    (b"x" * 4095 + b"\n", 2), (b"x" * 4096 + b"\n" + b"assert y\n", 1), (b"\n" * 5000, 2),
    (b"y" * 4090 + b"assert z == 1\nEXPECT_TRUE(q);\n", 1), (b"ASSERT_EQ(a,b);" * 1000, 2),
    (b"def test(self):\n" * 700, 1), (b"\x00\x01\xff\xfeassert\x80\n\x00", 1),
    (b"  \t  assert   x  ==  1   \t \n", 1), (b"self.assertEqual\n", 1), (b"EXPECT_\n", 2),
    (b"a" * 8200 + b" assert not x\n" + b"b" * 100 + b"\n", 1),
    (b"no newline at end assert x < 1", 1), (PY_SAMPLE, 1), (CC_SAMPLE, 2), (JAVA_SAMPLE, 4),
    (CC_SAMPLE, 3), (CC_SAMPLE, 5), (CC_SAMPLE, 6), (PY_SAMPLE, 0), (CC_SAMPLE, 1), (PY_SAMPLE, 2),
]

TOKENS = [b"assert", b"ASSERT_", b"Assert", b"assert ", b"EXPECT_", b"EXPECT_EQ", b"expect_", b"test", b"Test", b"TEST",
          b"TEST_F", b"TEST_F(", b"def", b"def ", b"class", b"class ", b"class\t", b"void", b"{", b"}", b"(", b")", b"self.",
          b"assertEqual", b"assertTrue", b"assert_", b"assert_called_with", b"assertFoo", b" not ", b" in ", b" is not ",
          b"True", b"==", b"!=", b"<=", b">=", b"<", b">", b"not ", b" ", b"  ", b"\t", b"\r", b"x", b"y", b"_", b".", b",",
          b"EQ", b"NE", b"NEAR", b"FLOAT_EQ", b"DOUBLE_EQ", b"THROW", b"STREQ", b"//", b"#", b'"', b"asser", b"ssert",
          b"EXPECT", b"tes", b"clas", b"voi", b"de", b"\x00", b"\xc3\xa9", b"0", b"9", b"assertassert", b"testtest",
          b"BOOST_CHECK", b"BOOST_CHECK_EQUAL", b"BOOST_CHECK(", b"NTA_CHECK(", b"TESTEQUAL", b"FAIL", b"_CHECK", b"_CHEC", b"TESTEQUA",
          b"!", b"(!", b"assert (", b"F", b"TEST_"]


def fuzz_file(rng: random.Random, size: int, nl_rate=0.08, long_lines=False, binary=False) -> bytes:
    """binary=True: every byte value, CRs in one draw of eight, and runs of 0xFF / 0x00 (the Mersenne-61 hash edges of
    SPEC section 3) between the tokens."""
    out = bytearray()
    while len(out) < size:
        r = rng.random()
        if r < nl_rate:
            out += b"\n"
        elif r < nl_rate + 0.02 and long_lines:
            out += bytes(rng.choice(b"abcdefgxyz ._(") for _ in range(rng.randrange(200, 6000)))
        elif binary and r < nl_rate + 0.15:
            out += b"\r"
        elif binary and r < nl_rate + 0.45:
            out += bytes([rng.randrange(256)])
        elif binary and r < nl_rate + 0.5:
            out += bytes([rng.choice((0x00, 0xFF))]) * rng.randrange(1, 20)
        else:
            out += rng.choice(TOKENS)
    out = bytes(out[:size])
    if rng.random() < 0.5 and out and not out.endswith(b"\n"):
        out = out[:-1] + b"\n"
    return out


def fuzz_corpus(seed: int, n_files: int, max_size: int, long_lines=False, binary=False):
    rng = random.Random(seed)
    files, exts = [], []
    for i in range(n_files):
        kind = rng.random()
        if kind < 0.1:
            size = rng.randrange(0, 40)
        elif kind < 0.2:
            size = rng.choice([4095, 4096, 4097, 8191, 8192, 8193, 4096 + 239, 4096 + 240, 4096 + 241, 12288])
            size = min(size, max_size)
        else:
            size = rng.randrange(1, max_size)
        files.append(fuzz_file(rng, size, nl_rate=rng.choice([0.01, 0.05, 0.1, 0.3]), long_lines=long_lines, binary=binary))
        exts.append(rng.choice([0, 1, 1, 2, 2, 3, 4, 5, 6]))
    grps = [rng.randrange(0, 5) for _ in range(n_files)]
    return files, np.array(exts, np.uint8), np.array(grps, np.uint16)


M61 = (1 << 61) - 1


def cr_wrap_content(rng: random.Random, n: int) -> bytes:
    """n >= 8 bytes without LF whose value N (SPEC section 3) makes the line `content + CR` hash to
    (N + 13 * 256^n) mod (2^61 - 1) below 13 * 256^n mod (2^61 - 1): dropping the CR has to wrap around the modulus.
    (Below 8 bytes N + 13 * 256^n < 2^61 - 1 and it cannot.)  The top bytes are random; the low 8 pick the residue."""
    cr = 13 * pow(256, n, M61) % M61
    while True:
        high = bytes(rng.choice(range(11, 256)) for _ in range(n - 8))
        r = M61 - 1 - rng.randrange(cr)                  # N mod p in [p - cr, p)
        low = (r - 8 * int.from_bytes(high, "little")) % M61   # 256^8 = 2^64 = 8 mod 2^61 - 1
        c = low.to_bytes(8, "little") + high
        if b"\n" not in c:
            return c


def hash_edge_contents(seed=5):
    """Line contents at the edges of the Mersenne-61 line hash: 0xFF runs (every byte 2^8 - 1, values >= 2^61), multiples
    of 2^61 - 1 (value 0 mod p, also with zero bytes behind), CR steps that wrap, zero bytes and bare CRs."""
    rng = random.Random(seed)
    out = [b"\xff" * n for n in range(1, 301)]
    for k in range(1, 40):
        v = (k * M61).to_bytes((k * M61).bit_length() // 8 + 1, "little")
        out += [c for c in (v, v + b"\x00", v + b"\x00" * 5) if b"\n" not in c]
    out += [cr_wrap_content(rng, n) + b"\r" for n in range(8, 301, 2)]
    out += [b"\x00" * n for n in (1, 2, 7, 8, 9, 15, 16, 17, 61, 62, 300)]
    out += [b"\r", b"\r\r", b"x\r\r", b"\xff" * 8 + b"\r", b"\x00\r"]
    return out


def table_name_variants(names):
    """Each category table name and its near misses: one byte flipped, dropped or appended at every position, a
    prefix, and cuts / extensions to the lengths around the 8- and 16-byte load boundaries of the device lookup."""
    out = []
    for nm in names:
        out.append(nm)
        for i in range(len(nm)):
            out.append(nm[:i] + bytes([nm[i] ^ 0x20 if nm[i] != 0x5F else 0x41]) + nm[i + 1:])
            out.append(nm[:i] + nm[i + 1:])
        out += [nm + b"x", nm + b"_", nm + b"0", b"x" + nm, b"my_" + nm, b"_" + nm]
        out += [nm[:k] for k in (6, 7, 8, 9, 15, 16, 17) if k < len(nm)]
        out += [nm + b"q" * (k - len(nm)) for k in (8, 9, 16, 17, 24) if k > len(nm)]
    return list(dict.fromkeys(out))


def edge_corpus():
    files = [f for f, _ in EDGE_FILES]
    exts = np.array([e for _, e in EDGE_FILES], np.uint8)
    grps = np.array([i % 3 for i in range(len(files))], np.uint16)
    return files, exts, grps


def load_fixture(path):
    """Files of a tests/golden/*.npz corpus fixture (tools/make_golden.py: c1_fixture, c1_hazards)."""
    d = np.load(path)
    blob, size = d["blob"], d["size"].astype(np.int64)
    ends = np.cumsum(size)
    files = [blob[e - s:e].tobytes() for s, e in zip(size, ends)]
    grps = d["grp"].astype(np.uint16)
    return files, d["ext"].astype(np.uint8), grps, int(grps.max()) + 1 if len(grps) else 1


def score_g1(golden, names, files, events):
    """Golden G1 (ML-Testing-v1.xlsx!DeepSpeech rows of the bundled files): how many sheet statements the Rev-B events
    reproduce, and how much of their counts.  events: assertion events of a scan over `files`."""
    import collections
    by_file = collections.defaultdict(collections.Counter)
    for e in events:
        f = files[int(e["file"])]
        by_file[int(e["file"])][f[int(e["stmt_off"]):int(e["stmt_off"]) + int(e["stmt_len"])].decode("latin-1")] += 1
    idx = {n: i for i, n in enumerate(names)}
    stm, cnt, per_file = [0, 0], [0, 0], {}
    for name, want in golden.items():
        got = by_file[idx[name]]
        fs = fc = 0
        for st, (c, _) in want.items():
            stm[1] += 1
            cnt[1] += c
            if got.get(st):
                stm[0] += 1
                cnt[0] += min(c, got[st])
                fs += 1
                fc += min(c, got[st])
        per_file[name] = ([fs, len(want)], [fc, sum(c for c, _ in want.values())])
    return stm, cnt, per_file


def load_fixture_names(path):
    d = np.load(path)
    return bytes(d["names"]).decode().split("\n")


# ---------------------------------------------------------------------------------------------- revision pairs (SPEC section 8)
# Lines of the tie-heavy pairs: blank lines, braces, CR variants that hash like their LF twins, and assertion lines.
TIE_LINES = [b"\n", b"\r\n", b"}\n", b"}\r\n", b"  }\n", b"x\n", b"x\r\n", b"assert x\n", b"EXPECT_TRUE(ok);\n",
             b"self.assertEqual(a, b)\n", b"{\n"]


def tie_pair(rng: random.Random, n_lines: int, n_edits: int):
    """(old, new) over an alphabet of 2-4 lines: a random old file and n_edits random insertions, deletions and
    replacements of one line.  With so few distinct lines many alignments tie."""
    alpha = rng.sample(TIE_LINES, rng.randrange(2, 5))
    old = [rng.choice(alpha) for _ in range(n_lines)]
    new = list(old)
    for _ in range(n_edits):
        i = rng.randrange(len(new) + 1)
        op = rng.randrange(3)
        if op == 0 or not new:
            new.insert(i, rng.choice(alpha))
        elif op == 1 and i < len(new):
            del new[i]
        elif i < len(new):
            new[i] = rng.choice(alpha)
    o, n = b"".join(old), b"".join(new)
    if rng.random() < 0.2 and o.endswith(b"\n"):          # an unterminated last line (equal to its terminated twin)
        o = o[:-1]
    return o, n


def tie_heavy_pairs(seed: int, scale: int = 1):
    """Tie-heavy pairs sized for every k_diff_small size and the left-over kernels: (olds, news, exts)."""
    rng = random.Random(seed)
    shapes = ([(rng.randrange(8, 200), rng.randrange(1, 12)) for _ in range(40)] +         # middle <= 512, D <= 31
              [(rng.randrange(300, 480), rng.randrange(12, 26)) for _ in range(16)] +     # <= 1 024 / 63
              [(rng.randrange(700, 1900), rng.randrange(10, 26)) for _ in range(10)] +    # <= 4 096 / 63
              [(rng.randrange(700, 1900), rng.randrange(36, 56)) for _ in range(10)] +    # <= 4 096 / 127
              [(rng.randrange(2200, 2600), rng.randrange(4, 20)) for _ in range(5)] +     # middle > 4 096
              [(rng.randrange(300, 900), rng.randrange(90, 160)) for _ in range(5)])      # D > 127
    olds, news, exts = [], [], []
    for _ in range(scale):
        for n_lines, n_edits in shapes:
            o, n = tie_pair(rng, n_lines, n_edits)
            olds.append(o)
            news.append(n)
            exts.append(rng.choice((1, 2, 4)))
    return olds, news, exts


def block_pair(tag: bytes, old_blocks, new_blocks, n_prefix=3, n_suffix=2, assert_every=5):
    """A pair with a closed-form script: unique old blocks and unique new blocks (sizes old_blocks[i], new_blocks[i]; 0 =
    none) between unique common lines, behind a common prefix and before a common suffix.  The only LCS is the common
    lines, so every block pair is one hunk and every block line changes.  Every assert_every-th block line is an assertion
    line.  Returns (old, new, want) with want = (hunks_add, hunks_del, hunks_mod, deleted, inserted): line indices."""
    def blk(side, i, k):
        return [(b"assert %s_%s%d_%d\n" if j % assert_every == 1 else b"%s_%s%d_%d = 1\n") % (tag, side, i, j) for j in range(k)]
    old = [b"%s_pre%d\n" % (tag, i) for i in range(n_prefix)]
    new = list(old)
    deleted, inserted, h = [], [], [0, 0, 0]
    for i, (ko, kn) in enumerate(zip(old_blocks, new_blocks)):
        deleted += range(len(old), len(old) + ko)
        inserted += range(len(new), len(new) + kn)
        old += blk(b"o", i, ko)
        new += blk(b"n", i, kn)
        if ko or kn:
            h[2 if ko and kn else 0 if kn else 1] += 1
        common = [b"%s_common%d\n" % (tag, i)]
        old += common
        new += common
    tail = [b"%s_suf%d\n" % (tag, i) for i in range(n_suffix)]
    return b"".join(old + tail), b"".join(new + tail), (h[0], h[1], h[2], deleted, inserted)
