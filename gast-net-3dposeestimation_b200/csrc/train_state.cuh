// Saved-for-backward state of one training forward (see train.cuh).
#pragma once
#include <string>
#include <vector>
#include "gast_common.cuh"

using gast::RowMap;

// Schedule of a model forward, decided by geometry() (gast_api.cu).
struct StageGeo {            // one temporal stage
  int taps = 0, dil = 1, stride = 1;
  int Tin = 0, Tout = 0;     // frames per clip in and out
  RowMap tapmap, resmap;     // output frame -> input frame of its first tap / of its residual
};

struct Geometry {
  int T0 = 0;                // frames per clip after the expand conv
  int s0 = 1;                // stride of the expand conv (filter width when strided, else 1)
  std::vector<StageGeo> stages;   // stage i at index i-1
  int T_out = 0;
};

struct BnSave {
  const float* Z = nullptr; int ldz = 0; long long M = 0; int N = 0;
  float* mean = nullptr; float* invstd = nullptr;
  const float* gamma = nullptr; const float* beta = nullptr;
  int relu = 0; const unsigned char* keep = nullptr; float kscale = 1.f;
  bool frozen = false;   // mean / invstd are the running statistics (eval-mode BatchNorm)
  std::string prefix;
};

struct BlockSave {
  int C = 0; long long F = 0;
  const float* X = nullptr;
  float *Wst = nullptr, *H = nullptr, *coefA[2] = {nullptr, nullptr}, *S = nullptr, *XY = nullptr, *Zlc = nullptr, *L = nullptr;
  float *G = nullptr, *AB = nullptr, *Y = nullptr, *Zgc = nullptr, *Gl = nullptr, *Zbc = nullptr, *Out = nullptr;
  BnSave bn1, bn2, bnlc, bngc, bnbc;
  std::string P;
};

struct StageSave {
  StageGeo g; int Cw = 0;
  const float* X = nullptr; float *Wt = nullptr, *Z1 = nullptr, *Hh = nullptr, *Z2 = nullptr, *Out = nullptr;
  BnSave bnA, bnB;
  int idx = 0;
};

struct TrainState {
  bool valid = false;
  // frozen: the eval-mode forward (model.eval()) -- BatchNorm on the running statistics, which stay untouched, no
  // dropout, and the schedule `sn` of gast_forward (strided_now); otherwise train mode on the handle's own schedule
  bool frozen = false; int sn = 0;
  int B = 0, T = 0;
  Geometry geo;
  const float* x = nullptr;
  float *xbn = nullptr, *Acol = nullptr, *We8 = nullptr, *Z0 = nullptr, *act0 = nullptr;
  BnSave bnin, bnex;
  std::vector<BlockSave> blocks;
  std::vector<StageSave> stages;
  const float* last = nullptr;   // input of shrink
  // partials area of every column reduction of the forward and its backward (col_partials), in the forward's part of
  // the workspace
  double* red_part = nullptr;
  float drop_p = 0.f; unsigned long long seed = 0; unsigned long long drop_ctr = 0;
  size_t arena_off = 0;          // workspace used by the forward (backward temporaries go after it)
  size_t workspace_bytes = 0;    // what the forward checked: its own sizing pass plus a backward with parameter gradients,
                                 // which bounds every backward of it
};

