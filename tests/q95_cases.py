"""Quality 9.5 (BROTLI_PARAM_Q9_5) configurations shared by tests/test_model_q95.py (CPU model, sha256 goldens) and
tests/test_gpu_q95.py (device == the same goldens).

With Q9_5 quality 10 parses with H9 and quality 11 with H5 / H6 at bucket depth 512 (H6 when the size hint is above 1 MiB and
lgwin >= 19; lgwin <= 16 takes H6 at depth 256), both greedy / lazy; the metablocks are built as at quality 10 / 11.  The
cases cover alice29, 6 MB of text and JSON logs (>= 4 MiB: the parse searches the buckets on demand), lgwin 16 / 22 / 24,
size hints on both sides of 1 MiB and 4 MiB, the static dictionary off, literal context modelling off, and a 17 MB input at
lgwin 24, whose chunk takes two sort batches."""
import hashlib
import os

MIB = 1 << 20
_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# name: (input, quality, lgwin, size hint (0 = input size), encoder options (CPU model field names))
CASES = {
    "alice-q10-w22": ("alice", 10, 22, 0, {}),
    "alice-q11-w22": ("alice", 11, 22, 0, {}),
    "alice-q10-w16": ("alice", 10, 16, 0, {}),
    "alice-q11-w16": ("alice", 11, 16, 0, {}),
    "alice-q11-w24": ("alice", 11, 24, 0, {}),
    "alice-q11-hint-1MiB": ("alice", 11, 22, MIB, {}),
    "alice-q11-hint-1MiB+1": ("alice", 11, 22, MIB + 1, {}),
    "alice-q11-hint-4MiB": ("alice", 11, 22, 4 * MIB, {}),
    "alice-q11-hint-4MiB+1": ("alice", 11, 22, 4 * MIB + 1, {}),
    "alice-q11-no-dict": ("alice", 11, 22, 0, {"use_dict": 0}),
    "alice-q10-no-ctx": ("alice", 10, 22, 0, {"ctx_model": 0}),
    "text6-q11-w22": ("text6", 11, 22, 0, {}),
    "text6-q11-hint-1MiB": ("text6", 11, 22, MIB, {}),
    "text6-q10-w22": ("text6", 10, 22, 0, {}),
    "json6-q10-w22": ("json6", 10, 22, 0, {}),
    "json6-q11-hint-4MiB": ("json6", 11, 22, 4 * MIB, {}),
    "json6-q11-no-ctx": ("json6", 11, 22, 0, {"ctx_model": 0}),
    "json6-q11-no-dict": ("json6", 11, 22, 0, {"use_dict": 0}),
    "text17-q11-w24": ("text17", 11, 24, 0, {}),
}

# sha256 of the CPU model's stream of each case
GOLDEN = {
    "alice-q10-w22": "36b1eee3c7791baf65b8cb100241a677bfa00c2a862a38a5268e6897a63d6fef",
    "alice-q11-w22": "78b9b8d07ecd5eacb40d9af0a59bc7b261710f757f9a797bffe83855e14326a5",
    "alice-q10-w16": "b29d6a9cbc035d36bcc4949dc97c270066f8b245f6e02712f41d012f328689b8",
    "alice-q11-w16": "1b173e0f36730af26ec2257098b2f27c57ec067e923f43bfff3163fb8f436cc3",
    "alice-q11-w24": "902e203569de66e9d0bd1554d3942932d5feb2b5dcdfa26cbb4d736c2cca6769",
    "alice-q11-hint-1MiB": "78b9b8d07ecd5eacb40d9af0a59bc7b261710f757f9a797bffe83855e14326a5",
    "alice-q11-hint-1MiB+1": "8e3e740b2580f4c129e2f0222ba2aa243025959f5a1fe4626a3808f675e94460",
    "alice-q11-hint-4MiB": "8e3e740b2580f4c129e2f0222ba2aa243025959f5a1fe4626a3808f675e94460",
    "alice-q11-hint-4MiB+1": "8e3e740b2580f4c129e2f0222ba2aa243025959f5a1fe4626a3808f675e94460",
    "alice-q11-no-dict": "91d45e27c1d52e0b84044c19a195246dc5c556659b5c3bba523e40634f0fa0aa",
    "alice-q10-no-ctx": "1ccdaca24128aced6be8484086c9c37c8819f1d1141c1ba40ef64ec24bc95775",
    "text6-q11-w22": "a8c2bcf6ae12624769bc935f0e555185ca34706ec86285acc50645acccaf115e",
    "text6-q11-hint-1MiB": "41ae6f6f5aa04327f2cb105b82ef70877bd9ec2e1ced371916464988ef5633ab",
    "text6-q10-w22": "119604011a65dece016ddd596b5b7772341f29134c6ae4c6a09f9897cb941cc6",
    "json6-q10-w22": "b883b1f6dafef77d82601410458647d136425fa4c378400cf471d5b80ae21244",
    "json6-q11-hint-4MiB": "5ceee729b1fc411b729457d315f33b1443eb355018a1737748fafafdab54a944",
    "json6-q11-no-ctx": "cefbc78896fa8a1dfbced50a788d5b1330e6f85a0672ba38d9e9dc32f79e584a",
    "json6-q11-no-dict": "c41590c7054c6e91741b52459c16ad0191058af43976ffe891028c5dd8bd0f33",
    "text17-q11-w24": "7711f4c62110ed7ef033c605e1ff09eb62b1444aa081c9f4e23898f57a968846",
}


def hasher_q95(quality, lgwin, size_hint):
    """ChooseHasher with Q9_5 (encode.rs:834-893) as (hasher, key bits, depth), in the form of tests/match_ref.py's config:
    quality 10 takes H9; quality 11 falls through to the q5..q9 rules with block_bits = min(q - 1, 9); H6 is chosen above a
    1 MiB size hint instead of 4 MiB; H40..H42 of lgwin <= 16 run as H6 with depth 256 in this library."""
    q = min(max(quality, 5), 11)
    lgwin = min(max(lgwin, 10), 24)
    hint = min(size_hint, 0xFFFFFFFF)
    if q in (9, 10):
        return 9, 15, 256
    if lgwin <= 16:
        return 6, 15, 256
    if hint > 1 << 20 and lgwin >= 19:
        return 6, 15, 1 << min(q - 1, 9)
    return 5, 14 if q < 7 and hint <= 1 << 20 else 15, 1 << min(q - 1, 9)


def inputs(name):
    from tools import datagen
    if name == "alice":
        with open(os.path.join(_ROOT, "tests", "golden", "alice29.txt"), "rb") as f:
            return f.read()
    if name == "text6":
        return datagen.enwik_like(6_000_000)
    if name == "json6":
        return datagen.json_logs(6_000_000)
    if name == "text17":
        return datagen.enwik_like(17_000_000, seed=6)
    raise KeyError(name)


def sha(b):
    return hashlib.sha256(b).hexdigest()
