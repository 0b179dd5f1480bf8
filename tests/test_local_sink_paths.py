"""CPU tests for the local sink: Go's filepath.Join / Clean as sink.append_posts_grouped builds posts.jsonl paths (the
examples of the Go documentation for path/filepath on Unix), and the tgi_channel_appends structs against the header."""
import ctypes as C
import os
import subprocess
import tempfile

import pytest

from distributed_crawler_b200 import abi, sink

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("path, want", [
    (b"a/c", b"a/c"), (b"a//c", b"a/c"), (b"a/c/.", b"a/c"), (b"a/c/b/..", b"a/c"), (b"/../a/c", b"/a/c"),
    (b"/../a/b/../././/c", b"/a/c"), (b"", b"."), (b"//a", b"/a"), (b"///a/", b"/a"), (b"../../x", b"../../x"),
    (b"a/../..", b".."), (b"/", b"/"), (b"./", b"."),
])
def test_go_clean(path, want):
    assert sink.go_clean(path) == want


@pytest.mark.parametrize("elems, want", [
    ((b"a", b"b", b"c"), b"a/b/c"), ((b"a", b"b/c"), b"a/b/c"), ((b"a/b", b"c"), b"a/b/c"), ((b"a/b", b"/c"), b"a/b/c"),
    ((b"a/b", b"../../../xyz"), b"../xyz"), ((b"", b""), b""), ((b"a", b""), b"a"), ((b"", b"a"), b"a"),
    ((b"/srv/crawls", b"crawl-7", b"", b"posts"), b"/srv/crawls/crawl-7/posts"),  # an empty channelID drops out
    ((b"base/", b"crawl", b"chan_1", b"posts"), b"base/crawl/chan_1/posts"),
])
def test_go_join(elems, want):
    assert sink.go_join(*elems) == want


def test_channel_appends_structs_match_header():
    probe = r'''
#include <stdio.h>
#include <stddef.h>
#include "tgingest.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu %zu %zu\n", sizeof(tgi_channel_group), offsetof(tgi_channel_group, n_lines),
         offsetof(tgi_channel_group, byte_len), sizeof(tgi_channel_appends_t), offsetof(tgi_channel_appends_t, order),
         offsetof(tgi_channel_appends_t, kernel_ms), offsetof(tgi_channel_appends_t, gpu_launches));
  return 0;
}'''
    with tempfile.TemporaryDirectory() as d:
        src = os.path.join(d, "p.c")
        with open(src, "w") as f:
            f.write(probe)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), src, "-o", os.path.join(d, "p")])
        got = list(map(int, subprocess.check_output([os.path.join(d, "p")]).decode().split()))
    G, A = abi.CHANNEL_GROUP, abi.ChannelAppendsC
    assert got == [G.itemsize, G.fields["n_lines"][1], G.fields["byte_len"][1], C.sizeof(A), A.order.offset,
                   A.kernel_ms.offset, A.gpu_launches.offset]
