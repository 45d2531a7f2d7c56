// Online speaker clustering handle (dg_cluster_*), including the shared-identity records.
#include <memory>

#include "host.cuh"

extern "C" int dg_cluster_create(int max_speakers, int dim, double tau, double rho, double delta, int device,
                                 dg_cluster** out) {
  if (!out || max_speakers < 1 || max_speakers > 32 || dim < 1) {
    set_error("dg_cluster_create: need 1 <= max_speakers <= 32 and dim >= 1");
    return DG_EINVAL;
  }
  DG_CUDA(cudaSetDevice(device));
  std::unique_ptr<dg_cluster> h(new dg_cluster());
  h->device = device;
  h->p.M = max_speakers;
  h->p.D = dim;
  // numpy compares a float32 array with a Python float in float32 (weak scalar promotion)
  h->p.tau_f = (float)tau;
  h->p.rho_f = (float)rho;
  h->p.delta = delta;
  h->p.metric = 0;
  if (h->centers.ensure((size_t)max_speakers * dim * 8) || h->active.ensure(32 * 4) || h->init.ensure(2 * 4) ||
      h->base.ensure((size_t)max_speakers * dim * 8) || h->base_active.ensure(32 * 4) || h->relabel.ensure(32 * 4))
    return DG_ECUDA;
  *out = h.release();
  return DG_OK;
}

extern "C" int dg_cluster_set_metric(dg_cluster* h, int metric) {
  if (!h || metric < 0 || metric > 4) {
    set_error("dg_cluster_set_metric: 0 cosine, 1 euclidean, 2 sqeuclidean, 3 cityblock, 4 chebyshev");
    return DG_EINVAL;
  }
  h->p.metric = metric;
  return DG_OK;
}

extern "C" int dg_cluster_step(dg_cluster* h, const float* seg, const float* emb, int B, int F, int K, int32_t* map,
                               float* permuted, void* stream) {
  if (!h || !seg || !emb || !map || B < 0 || F < 1 || K < 1) {
    set_error("dg_cluster_step: bad arguments");
    return DG_EINVAL;
  }
  DG_CUDA(cudaSetDevice(h->device));
  if (h->prep.ensure(cluster_prep_floats(B, K) * 4 + 16) || h->prep_d.ensure(cluster_prep_doubles(B, K) * 8 + 16))
    return DG_ECUDA;
  return launch_cluster_step(h->p, seg, emb, B, F, K, h->centers.as<double>(), h->active.as<int>(),
                             h->init.as<int>(), h->prep.as<float>(), h->prep_d.as<double>(), map, permuted,
                             (cudaStream_t)stream);
}

extern "C" int dg_cluster_reset(dg_cluster* h) {
  if (!h) return DG_EINVAL;
  DG_CUDA(cudaSetDevice(h->device));
  DG_CUDA(cudaDeviceSynchronize());
  DG_CUDA(cudaMemset(h->centers.p, 0, h->centers.bytes));
  DG_CUDA(cudaMemset(h->active.p, 0, h->active.bytes));
  DG_CUDA(cudaMemset(h->init.p, 0, h->init.bytes));
  DG_CUDA(cudaMemset(h->base.p, 0, h->base.bytes));
  DG_CUDA(cudaMemset(h->base_active.p, 0, h->base_active.bytes));
  return DG_OK;
}

extern "C" int dg_cluster_get_state(dg_cluster* h, double* centers, int32_t* active, int* initialized) {
  if (!h) return DG_EINVAL;
  DG_CUDA(cudaSetDevice(h->device));
  DG_CUDA(cudaDeviceSynchronize());
  int init[2] = {0, 0};
  DG_CUDA(cudaMemcpy(init, h->init.p, 8, cudaMemcpyDeviceToHost));
  if (init[1]) {
    set_error("Cannot update unknown centers");   // reference clustering.py:98 (AssertionError)
    return DG_EINVAL;
  }
  if (centers) DG_CUDA(cudaMemcpy(centers, h->centers.p, (size_t)h->p.M * h->p.D * 8, cudaMemcpyDeviceToHost));
  if (active) DG_CUDA(cudaMemcpy(active, h->active.p, (size_t)h->p.M * 4, cudaMemcpyDeviceToHost));
  if (initialized) *initialized = init[0];
  return DG_OK;
}

extern "C" int dg_cluster_set_state(dg_cluster* h, const double* centers, const int32_t* active, int initialized) {
  if (!h || !centers || !active) return DG_EINVAL;
  DG_CUDA(cudaSetDevice(h->device));
  DG_CUDA(cudaDeviceSynchronize());
  int init[2] = {initialized ? 1 : 0, 0};
  DG_CUDA(cudaMemcpy(h->centers.p, centers, (size_t)h->p.M * h->p.D * 8, cudaMemcpyHostToDevice));
  DG_CUDA(cudaMemcpy(h->active.p, active, (size_t)h->p.M * 4, cudaMemcpyHostToDevice));
  DG_CUDA(cudaMemcpy(h->init.p, init, 8, cudaMemcpyHostToDevice));
  DG_CUDA(cudaMemcpy(h->base.p, centers, (size_t)h->p.M * h->p.D * 8, cudaMemcpyHostToDevice));
  DG_CUDA(cudaMemcpy(h->base_active.p, active, (size_t)h->p.M * 4, cudaMemcpyHostToDevice));
  return DG_OK;
}

extern "C" int dg_cluster_destroy(dg_cluster* h) {
  delete h;
  return DG_OK;
}

// shared-identity extension (SURVEY.md 8(e), BASELINE config 5); kernels and rule in cluster.cu
extern "C" int dg_cluster_record_len(const dg_cluster* h) { return h ? h->p.M * h->p.D + h->p.M + 2 : 0; }

extern "C" int dg_cluster_export_delta(dg_cluster* h, double* record_dev, void* stream) {
  if (!h || !record_dev) {
    set_error("dg_cluster_export_delta: bad arguments");
    return DG_EINVAL;
  }
  DG_CUDA(cudaSetDevice(h->device));
  return launch_cluster_export(h->centers.as<double>(), h->active.as<int>(), h->base.as<double>(),
                               h->base_active.as<int>(), h->p.M, h->p.D, record_dev, (cudaStream_t)stream);
}

extern "C" int dg_cluster_merge(dg_cluster* h, const double* records_dev, int world, int rank, int32_t* maps_dev,
                                int n_maps, void* stream) {
  if (!h || !records_dev || world < 1 || rank < 0 || rank >= world) {
    set_error("dg_cluster_merge: bad arguments");
    return DG_EINVAL;
  }
  DG_CUDA(cudaSetDevice(h->device));
  int rc;
  if ((rc = launch_cluster_merge(records_dev, world, rank, h->p, dg_cluster_record_len(h), h->centers.as<double>(),
                                 h->active.as<int>(), h->base.as<double>(), h->base_active.as<int>(),
                                 h->init.as<int>(), h->relabel.as<int32_t>(), (cudaStream_t)stream)))
    return rc;
  if (maps_dev && n_maps > 0) return launch_relabel_maps(maps_dev, n_maps, h->relabel.as<int32_t>(), (cudaStream_t)stream);
  return DG_OK;
}
