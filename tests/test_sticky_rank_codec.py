"""The outcome byte of a step the speculative pass accepted as sticky (blance_b200/csrc/sticky_rank.cuh): the
scouts pack the (score, position) ranks of the step's current nodes, the leader stores them next to the "accepted"
flag in one byte, and k_scatter_stream writes the nodes back in rank order.  A host program built with nvcc from
the same header runs every permutation of ranks for k = 1..4, with the scout's word around the ranks as the kernel
builds it (generation above, node below), and checks that the byte is flagged, that the decoded row is the current
nodes in rank order and that every output slot is written exactly once.  The same program built with all four
ranks packed - the layout in which node 3's high rank bit is the flag - must fail.  CPU only."""
import os
import shutil
import subprocess
import tempfile

import pytest

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "blance_b200", "csrc")
NVCC = os.environ.get("NVCC", shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc")

SRC = r'''
#include <algorithm>
#include <cstdio>
#include "sticky_rank.cuh"
using namespace blance_dev;

template <int K> static long check() {
  int rank[K];                       // rank[q] = rank of current node q
  for (int q = 0; q < K; ++q) rank[q] = q;
  long bad = 0;
  do {
    int32_t nodes[K];
    for (int q = 0; q < K; ++q) nodes[q] = 1000 + 7 * q;
    for (uint32_t gen : {0u, 0x3FFu}) {
      for (uint32_t tp : {0u, 0x1FFFu}) {
        uint32_t ranks = 0;          // the scout (assign_pass_spec.cuh): z = gen << 21 | ranks << 13 | node
        for (int q = 0; q < K; ++q) ranks = srank_pack<K>(ranks, q, rank[q]);
        const uint32_t z = (gen << 21) | (ranks << 13) | tp;
        const uint8_t b = srank_byte(z >> 13);   // the leader
        if (!srank_accepted(b)) ++bad;
        int32_t out[8];
        std::fill(out, out + 8, -1);
        srank_expand<K>(b, nodes, out);          // k_scatter_stream
        int writes[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        int below = 0;
        for (int q = 0; q < K; ++q) {
          const int r = srank_rank<K>(b, q, below);
          below += r;
          if (r < 0 || r >= 8) { ++bad; continue; }
          ++writes[r];
        }
        for (int r = 0; r < 8; ++r) if (writes[r] != (r < K ? 1 : 0)) ++bad;
        for (int q = 0; q < K; ++q) if (out[rank[q]] != nodes[q]) ++bad;
        for (int r = K; r < 8; ++r) if (out[r] != -1) ++bad;
      }
    }
  } while (std::next_permutation(rank, rank + K));
  return bad;
}

int main() {
  std::printf("%ld %ld %ld %ld\n", check<1>(), check<2>(), check<3>(), check<4>());
  return 0;
}
'''


def run_codec(*defines):
    if not os.path.exists(NVCC):
        pytest.skip("nvcc is not available")
    with tempfile.TemporaryDirectory() as d:
        src = os.path.join(d, "codec.cu")
        open(src, "w").write(SRC)
        exe = os.path.join(d, "codec")
        subprocess.run([NVCC, "-std=c++17", "-O1", "-I" + CSRC, *defines, src, "-o", exe], check=True)
        return [int(x) for x in subprocess.run([exe], stdout=subprocess.PIPE, text=True, check=True).stdout.split()]


def test_every_rank_permutation_round_trips_for_k_1_to_4():
    assert run_codec() == [0, 0, 0, 0]


def test_packing_all_four_ranks_is_caught():
    # bit 7 is then both the flag and node 3's high rank bit: k = 1..3 still decode, k = 4 does not
    bad = run_codec("-DBL_SRANK_PACKED=4")
    assert bad[:3] == [0, 0, 0] and bad[3] > 0
