// talkshow_b200 — packed conv stacks of the body path (see convstack.cu).
#pragma once
#include "kernels.h"

namespace ts {

struct ResStack {
  Layer l0, l1, fin;
};

struct Trunk {  // AudioEncoder / VQ Encoder trunk
  int in_dim = 0, hid = 0;
  Layer project, down1, down2;
  ResStack s1, s2, s3;
};

struct VQNet {
  bool loaded = false;
  int out_dim = 0, ncodes = 0;
  Trunk enc;
  Layer pre_vq, aft_vq, project;
  Layer up2e, up2o, up3e, up3o;
  ResStack d1, d2, d3;
  float* codebook = nullptr;  // [ncodes][64]
  float* ee = nullptr;        // [ncodes] squared norms
};

struct ConvStacks {
  bool audio_loaded = false;
  Trunk audio;
  VQNet vq[2];
};

void pack_trunk(ts_engine* e, const Ckpt& ck, const std::string& p, int in_dim, int hid, Trunk* t);
void pack_vq(ts_engine* e, const Ckpt& ck, VQNet* v);
Act3 new_act(ts_engine* e, int B, int T, int C, int pad, cudaStream_t s, bool split = false, int tail = 0, bool planes_only = false);
Act3 run_trunk(ts_engine* e, const Trunk& t, const Act3& x, cudaStream_t s);
Act3 run_decoder(ts_engine* e, const VQNet& v, const Act3& q, cudaStream_t s);
Act3 run_vq_decode(ts_engine* e, const VQNet& v, const int64_t* idx, int B, int T, cudaStream_t s);

// sizing pass + real pass over the same code path
template <class F>
void run_sized(ts_engine* e, F&& body) {
  e->ws.begin_sizing();
  body();
  size_t need = e->ws.need;
  e->ws.buf.ensure(need + 256);
  e->ws.begin(need);
  body();
}

}  // namespace ts
