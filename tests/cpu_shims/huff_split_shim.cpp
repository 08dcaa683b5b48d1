// Host build of the rules of the long-segment Huffman encoder (gj_hs_* in gpujpeg_b200/csrc/gj_device.cuh), for
// tests/test_huff_split_model.py.  Test infrastructure only.  Build: g++ -O2 -shared -fPIC.
#include <cstdint>

#include "../../gpujpeg_b200/csrc/gj_device.cuh"

extern "C" {

int hs_ff_count(uint32_t w) { return gj_hs_ff_count(w); }
uint32_t hs_stuffed_bytes(const uint32_t* w, uint32_t nbytes) { return gj_hs_stuffed_bytes(w, nbytes); }
void hs_image_words(const uint32_t* chunk, uint64_t stride, const uint64_t* e, int k, uint64_t w0, uint32_t n, uint32_t* out)
{
    gj_hs_image_words(chunk, stride, e, k, w0, n, out);
}
int hs_chunks(int blocks) { return gj_hs_chunks(blocks); }
uint64_t hs_tiles(uint64_t bits) { return gj_hs_tiles(bits); }
int hs_chunk_blocks() { return GJ_HS_CHUNK; }
int hs_tile_bytes() { return GJ_HS_TILE; }

uint32_t hs_keep(uint32_t nbytes) { return gj_hs_keep(nbytes); }
uint32_t hs_seg_front(int s, uint32_t pre) { return gj_hs_seg_front(s, pre); }
uint32_t hs_seg_back(int s, int segs, int last_of_frame) { return gj_hs_seg_back(s, segs, last_of_frame != 0); }
uint64_t hs_tiles_per_slot(uint64_t slot_stride) { return gj_hs_tiles_per_slot(slot_stride); }
uint64_t hs_status_words(int seg_count, int segblk, uint64_t slot_stride) { return gj_hs_status_words(seg_count, segblk, slot_stride); }
}
