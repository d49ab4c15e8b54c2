// CLI-compatible replacements of the reference's two native binaries, running the GPU solvers of
// libmvm_b200.so behind the reference's CSV file protocol (SURVEY.md §8 f-4):
//
//   bundle_adjuster <dir>   reads <dir>/ba_in.csv, writes <dir>/ba_out.csv
//                           (bundle_adjuster.cpp, ba_problem.cpp:8-113: the line type is decided by its field
//                           count -- 8 header, 3 point, 4..6 observation, 12 camera; result = 12 fields per
//                           camera, rotation column-major, 12 significant digits)
//   ba_initializer <dir>    reads <dir>/ba_init_in.csv, writes <dir>/ba_init_out.csv
//                           (ba_initializer.cpp, ba_init.cpp:10-75: 10 fields = view id + rotation, 14 fields =
//                           view pair + relative rotation + position of the second camera)
//
// Built twice from this file (-DMVM_CLI_BA_INIT selects ba_initializer).  The problems accepted are the ones
// the reference's writer emits (bundle_adjust_io.py:193-259): every 3-D point is observed exactly twice, by two
// different cameras (one weight per observation, equal in x and y), fx == fy, at most 8 cameras.  Anything else is refused with a
// message and a non-zero exit code -- there is no CPU fallback solver in here.
#include <cuda_runtime.h>

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <iomanip>
#include <iostream>
#include <map>
#include <string>
#include <vector>

#include "../../../include/mvm_b200.h"

namespace {

std::vector<std::string> split(const std::string& line, char sep) {
  std::vector<std::string> out;
  std::string cur;
  for (char c : line) {
    if (c == sep) { out.push_back(cur); cur.clear(); }
    else if (c != '\r' && c != '\n') cur.push_back(c);
  }
  out.push_back(cur);
  return out;
}

[[noreturn]] void die(const std::string& msg, int code = 2) {
  std::cerr << "mvm_b200: " << msg << std::endl;
  std::exit(code);
}

void cuda_ok(cudaError_t e, const char* what) {
  if (e != cudaSuccess) die(std::string(what) + ": " + cudaGetErrorString(e), 3);
}

template <class T>
struct DevBuf {
  T* p = nullptr;
  size_t n = 0;
  explicit DevBuf(size_t count) : n(count) { cuda_ok(cudaMalloc(&p, (count ? count : 1) * sizeof(T)), "cudaMalloc"); }
  DevBuf(const std::vector<T>& h) : DevBuf(h.size()) { upload(h); }
  ~DevBuf() { cudaFree(p); }
  void upload(const std::vector<T>& h) {
    if (!h.empty()) cuda_ok(cudaMemcpy(p, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice), "cudaMemcpy H2D");
  }
  std::vector<T> download() const {
    std::vector<T> h(n);
    if (n) cuda_ok(cudaMemcpy(h.data(), p, n * sizeof(T), cudaMemcpyDeviceToHost), "cudaMemcpy D2H");
    return h;
  }
};

void need_gpu() {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n < 1) die("no CUDA device: this binary only runs the sm_90a solvers", 3);
}

// 12 fields per camera: rotation column-major then translation (ba_problem.cpp:97-113, ba_init.cpp:58-75)
void write_cameras(const std::string& path, const std::vector<double>& extr, int n) {
  std::ofstream f(path);
  if (!f) die("cannot write " + path);
  for (int v = 0; v < n; ++v) {
    const double* E = extr.data() + (size_t)v * 16;
    for (int c = 0; c < 3; ++c)
      for (int r = 0; r < 3; ++r) f << std::setprecision(12) << E[r * 4 + c] << ",";
    f << std::setprecision(12) << E[3] << "," << E[7] << "," << E[11] << "\n";
  }
}

// all pairs a < b, ordered like the reference's loops (for b: for a < b)
void all_pairs(int T, std::vector<int>& pa, std::vector<int>& pb, std::map<std::pair<int, int>, int>& index) {
  for (int b = 1; b < T; ++b)
    for (int a = 0; a < b; ++a) {
      index[{a, b}] = (int)pa.size();
      pa.push_back(a);
      pb.push_back(b);
    }
}

#ifndef MVM_CLI_BA_INIT
int run_bundle_adjuster(const std::string& dir) {
  const std::string in_path = dir + "/ba_in.csv";
  std::ifstream file(in_path);
  if (!file) die("cannot read " + in_path);
  int n_cams = -1, fixed_cam = 0, n_pts = 0, n_obs = 0;
  double fx = 1, fy = 1, cx = 0, cy = 0;
  struct Ob { int cam, pt; double x, y, wx, wy; };
  std::vector<Ob> obs;
  std::vector<double> cams, pts;   // cams: 12 per camera as in the file
  std::string line;
  while (std::getline(file, line)) {
    const auto e = split(line, ',');
    if (e.size() == 8) {
      n_cams = std::stoi(e[0]); fixed_cam = std::stoi(e[1]); n_pts = std::stoi(e[2]); n_obs = std::stoi(e[3]);
      fx = std::stod(e[4]); fy = std::stod(e[5]); cx = std::stod(e[6]); cy = std::stod(e[7]);
    } else if (e.size() == 3) {
      for (int i = 0; i < 3; ++i) pts.push_back(std::stod(e[i]));
    } else if (e.size() >= 4 && e.size() <= 6) {
      Ob o{std::stoi(e[0]), std::stoi(e[1]), std::stod(e[2]), std::stod(e[3]), 1.0, 1.0};
      if (e.size() == 5) o.wx = o.wy = std::stod(e[4]);
      if (e.size() == 6) { o.wx = std::stod(e[4]); o.wy = std::stod(e[5]); }
      obs.push_back(o);
    } else if (e.size() == 12) {
      for (int i = 0; i < 12; ++i) cams.push_back(std::stod(e[i]));
    }
  }
  if (n_cams < 2) die("ba_in.csv: missing header or fewer than two cameras");
  if (n_cams > MVM_MAX_VIEWS) die("ba_in.csv: more than " + std::to_string(MVM_MAX_VIEWS) + " cameras is not supported");
  if ((int)cams.size() != 12 * n_cams) die("ba_in.csv: camera lines do not match the header");
  if ((int)pts.size() != 3 * n_pts || (int)obs.size() != n_obs) die("ba_in.csv: point / observation lines do not match the header");
  if (fixed_cam < 0 || fixed_cam >= n_cams) die("ba_in.csv: fixed camera out of range");
  if (std::fabs(fx - fy) > 1e-12 * std::fabs(fx) || fx == 0.0) die("ba_in.csv: fx != fy is not supported");

  // the solver keeps camera 0 fixed: swap labels fixed_cam <-> 0
  auto relabel = [&](int c) { return c == fixed_cam ? 0 : (c == 0 ? fixed_cam : c); };

  // every point must be seen exactly twice, by two different cameras, with one weight
  std::vector<int> first(n_pts, -1), second(n_pts, -1);
  for (int i = 0; i < n_obs; ++i) {
    const Ob& o = obs[i];
    if (o.pt < 0 || o.pt >= n_pts || o.cam < 0 || o.cam >= n_cams) die("ba_in.csv: observation index out of range");
    if (o.wx != o.wy) die("ba_in.csv: per-axis weights are not supported");
    if (first[o.pt] < 0) first[o.pt] = i;
    else if (second[o.pt] < 0) second[o.pt] = i;
    else die("ba_in.csv: a point with more than two observations is not supported (pairwise problems only)");
  }
  const int T = n_cams;
  std::vector<int> pa, pb;
  std::map<std::pair<int, int>, int> pidx;
  all_pairs(T, pa, pb, pidx);
  const int P = (int)pa.size();
  std::vector<std::vector<int>> members(P);   // point ids per pair, file order
  std::vector<char> flip(n_pts, 0);
  for (int k = 0; k < n_pts; ++k) {
    if (first[k] < 0 || second[k] < 0) die("ba_in.csv: a point with fewer than two observations is not supported");
    int ca = relabel(obs[first[k]].cam), cb = relabel(obs[second[k]].cam);
    if (ca == cb) die("ba_in.csv: both observations of a point in one camera");
    if (ca > cb) { std::swap(ca, cb); flip[k] = 1; }
    members[pidx[{ca, cb}]].push_back(k);
  }
  size_t n_max = 1;
  for (auto& m : members) n_max = std::max(n_max, m.size());
  const int n_pad = (int)((n_max + 63) / 64 * 64);

  std::vector<float> xa((size_t)P * n_pad * 2, 0.f), xb((size_t)P * n_pad * 2, 0.f), w((size_t)P * n_pad, 0.f),
      wb((size_t)P * n_pad, 0.f);
  std::vector<double> p0((size_t)P * n_pad * 3, 0.0);
  std::vector<int> n_valid(P, 0);
  for (int p = 0; p < P; ++p) {
    n_valid[p] = (int)members[p].size();
    for (size_t i = 0; i < members[p].size(); ++i) {
      const int k = members[p][i];
      const Ob& oa = obs[flip[k] ? second[k] : first[k]];
      const Ob& ob = obs[flip[k] ? first[k] : second[k]];
      const size_t o = (size_t)p * n_pad + i;
      // residual w (f X/Z + c - x) = (w f) (X/Z - (x - c)/f)
      xa[2 * o] = (float)((oa.x - cx) / fx); xa[2 * o + 1] = (float)((oa.y - cy) / fy);
      xb[2 * o] = (float)((ob.x - cx) / fx); xb[2 * o + 1] = (float)((ob.y - cy) / fy);
      w[o] = (float)(oa.wx * fx);      // one weight per observation (ba_problem.h:60-151)
      wb[o] = (float)(ob.wx * fx);
      for (int c = 0; c < 3; ++c) p0[3 * o + c] = pts[(size_t)3 * k + c];
    }
  }
  std::vector<double> extr((size_t)T * 16, 0.0);
  for (int v = 0; v < T; ++v) {
    const double* c = cams.data() + (size_t)12 * v;
    double* E = extr.data() + (size_t)relabel(v) * 16;
    for (int col = 0; col < 3; ++col)
      for (int r = 0; r < 3; ++r) E[r * 4 + col] = c[col * 3 + r];
    E[3] = c[9]; E[7] = c[10]; E[11] = c[11]; E[15] = 1.0;
  }

  need_gpu();
  DevBuf<float> d_xa(xa), d_xb(xb), d_w(w), d_wb(wb), d_out((size_t)T * 16);
  DevBuf<double> d_p0(p0), d_extr(extr), d_out64((size_t)T * 16), d_cost(2);
  DevBuf<int> d_nv(n_valid), d_it(1);
  const size_t ws_bytes = mvm_mvba_workspace_bytes(T, P, 1, n_pad);
  DevBuf<unsigned char> d_ws(ws_bytes);
  const int rc = mvm_multi_view_ba_obs(pa.data(), pb.data(), T, P, 1, n_pad, d_xa.p, d_xb.p, d_w.p, d_wb.p, d_nv.p, d_extr.p, d_p0.p,
                                      /*weights_prenormalized=*/1, d_out.p, d_out64.p, /*max_iterations=*/50, d_it.p,
                                      d_cost.p, d_ws.p, ws_bytes, nullptr);
  if (rc != 0) die("mvm_multi_view_ba_obs failed with status " + std::to_string(rc), 3);
  cuda_ok(cudaDeviceSynchronize(), "bundle adjustment kernel");
  const auto res = d_out64.download();
  const auto cost = d_cost.download();
  const auto iters = d_it.download();
  std::vector<double> out((size_t)T * 16);
  for (int v = 0; v < T; ++v)
    for (int i = 0; i < 16; ++i) out[(size_t)v * 16 + i] = res[(size_t)relabel(v) * 16 + i];
  write_cameras(dir + "/ba_out.csv", out, T);
  std::cout << "mvm_b200 bundle_adjuster: " << n_cams << " cameras, " << n_pts << " points, " << iters[0]
            << " iterations, cost " << cost[0] << " -> " << cost[1] << std::endl;
  return 0;
}
#else
int run_ba_initializer(const std::string& dir) {
  const std::string in_path = dir + "/ba_init_in.csv";
  std::ifstream file(in_path);
  if (!file) die("cannot read " + in_path);
  std::map<int, std::vector<double>> view_R;                       // id -> 9 column-major
  std::map<std::pair<int, int>, std::vector<double>> pair_Rp;      // (i,j) -> 9 column-major + position
  std::string line;
  while (std::getline(file, line)) {
    const auto e = split(line, ',');
    if (e.size() == 10) {
      std::vector<double> R(9);
      for (int i = 0; i < 9; ++i) R[i] = std::stod(e[i + 1]);
      view_R[std::stoi(e[0])] = R;
    } else if (e.size() == 14) {
      std::vector<double> v(12);
      for (int i = 0; i < 12; ++i) v[i] = std::stod(e[i + 2]);
      int i0 = std::stoi(e[0]), i1 = std::stoi(e[1]);
      if (i0 == i1) die("ba_init_in.csv: view pair with identical ids");
      if (i0 > i1) die("ba_init_in.csv: view pairs must be written with id0 < id1");
      pair_Rp[{i0, i1}] = v;
    }
  }
  const int T = (int)view_R.size();
  if (T < 2) die("ba_init_in.csv: fewer than two views");
  if (T > MVM_MAX_VIEWS) die("ba_init_in.csv: more than " + std::to_string(MVM_MAX_VIEWS) + " views is not supported");
  for (int v = 0; v < T; ++v)
    if (!view_R.count(v)) die("ba_init_in.csv: view ids must be 0..n-1");
  std::vector<int> pa, pb;
  std::map<std::pair<int, int>, int> pidx;
  all_pairs(T, pa, pb, pidx);
  const int P = (int)pa.size();
  std::vector<double> extr((size_t)T * 16, 0.0);
  for (int v = 0; v < T; ++v) {
    double* E = extr.data() + (size_t)v * 16;
    for (int col = 0; col < 3; ++col)
      for (int r = 0; r < 3; ++r) E[r * 4 + col] = view_R[v][col * 3 + r];
    E[15] = 1.0;
  }
  std::vector<float> T_rel((size_t)P * 16, 0.f);
  std::vector<unsigned char> present(P, 0);
  for (auto& kv : pair_Rp) {
    if (kv.first.first < 0 || kv.first.second >= T) die("ba_init_in.csv: view pair id out of range");
    const int p = pidx[kv.first];
    const auto& v = kv.second;
    float* M = T_rel.data() + (size_t)p * 16;
    double R[9];
    for (int col = 0; col < 3; ++col)
      for (int r = 0; r < 3; ++r) R[r * 3 + col] = v[col * 3 + r];
    for (int r = 0; r < 3; ++r) {
      for (int c = 0; c < 3; ++c) M[r * 4 + c] = (float)R[r * 3 + c];
      // file holds the position of camera id1 in camera id0's frame; T_rel carries t = -R position
      M[r * 4 + 3] = (float)(-(R[r * 3] * v[9] + R[r * 3 + 1] * v[10] + R[r * 3 + 2] * v[11]));
    }
    M[15] = 1.f;
    present[p] = 1;
  }
  need_gpu();
  DevBuf<double> d_extr(extr), d_out((size_t)T * 16);
  DevBuf<float> d_T(T_rel);
  DevBuf<unsigned char> d_present(present);
  DevBuf<int> d_edges(1);
  const int rc = mvm_ba_initialize(pa.data(), pb.data(), T, P, 1, 64, d_extr.p, d_T.p, d_present.p, d_present.p,
                                   /*inliers=*/nullptr, 0, d_out.p, d_edges.p, nullptr);
  if (rc != 0) die("mvm_ba_initialize failed with status " + std::to_string(rc), 3);
  cuda_ok(cudaDeviceSynchronize(), "ba_initialize kernel");
  write_cameras(dir + "/ba_init_out.csv", d_out.download(), T);
  std::cout << "mvm_b200 ba_initializer: " << T << " views, " << d_edges.download()[0] << " view pairs" << std::endl;
  return 0;
}
#endif

}  // namespace

int main(int argc, char** argv) {
#ifndef MVM_CLI_BA_INIT
  if (argc != 2) { std::cerr << "Usage: bundle_adjuster <path to read and write>\n"; return 1; }
  return run_bundle_adjuster(argv[1]);
#else
  if (argc != 2) { std::cerr << "Usage: ba_initializer <path to read and write>\n"; return 1; }
  return run_ba_initializer(argv[1]);
#endif
}
