/* ssb200.h -- C ABI of libssb200.so: the H100 (sm_90a) implementation of the
 * SoundSpaces per-step audio observation (binaural RIR (*) source -> waveform ->
 * log-magnitude spectrogram).
 *
 * The reference is 100 % Python and has no FFI of its own for this path; the
 * entry points below are what a ctypes binding inside the reference would bind
 * in place of the following reference code (paths relative to the upstream
 * repository, see INTEGRATION.md for the binding stub):
 *
 *   ssb_source_windows      <- the source-side half of scipy.signal.fftconvolve as
 *                              called at soundspaces/simulator.py:630,638,645,661 and
 *                              soundspaces/continuous_simulator.py:436,449 (one clip,
 *                              cached per (sound, sample offset) like
 *                              simulator.py:595-600 caches the decoded clip)
 *   ssb_convolve_batch      <- SoundSpacesSim._compute_audiogoal,
 *                              soundspaces/simulator.py:608-666 (all branches) and
 *                              ContinuousSoundSpacesSim._convolve_with_rir,
 *                              soundspaces/continuous_simulator.py:428-456
 *   ssb_crossfade_batch     <- crossfade(), soundspaces/continuous_simulator.py:47-53
 *   ssb_spectrogram_batch   <- SpectrogramSensor.compute_spectrogram,
 *                              soundspaces/tasks/nav.py:86-100
 *   ssb_render_batch        <- get_current_spectrogram_observation,
 *                              soundspaces/simulator.py:690-701 for a batch of envs
 *   ssb_render_batch_host   <- the same with host buffers (what the per-env numpy API
 *                              of the reference hands over), copies included
 *   ssb_sh_decode_batch     <- scripts/ambisonic_to_binaural.py:14-19 (closed AmbisonicBinauralizer ELF)
 *   ssb_sh_decode_multi_batch <- the same at orders 0 to 3 (1, 4, 9, 16 channels), every input at all of the
 *                              script's angles in one call
 *   ssb_intensity_batch     <- Intensity.get_observation, ss_baselines/av_wan/avwan_sensors.py:91-100
 *   ssb_audio_conv1_batch   <- permute(0, 3, 1, 2) + the first Conv2d + ReLU of AudioCNN,
 *                              ss_baselines/av_nav/models/audio_cnn.py:51-58,86 (rollout-time forward)
 *   ssb_audio_encoder_batch <- AudioCNN.forward under no_grad (rollout time): permute + the whole cnn Sequential,
 *                              ss_baselines/av_nav/models/audio_cnn.py:50-75,79-89, av_wan/models/audio_cnn.py:51-76,
 *                              savi/models/audio_cnn.py:61-92 without category channels
 *   ssb_audio_encoder_category_batch <- the same for SAVi with a distractor sound: permute + expand + cat of the
 *                              category observation + the whole cnn, savi/models/audio_cnn.py:135-150
 *   ssb_visual_encoder_batch <- VisualCNN.forward under no_grad (rollout time): permute + RGB / 255 + cat + the
 *                              whole cnn, ss_baselines/av_nav/models/visual_cnn.py:137-161, av_wan :95-118, savi :163-188
 *   ssb_map_encoder_batch   <- MapCNN.forward under no_grad (rollout time), AV-WaN's geometric and acoustic map
 *                              encoders: permute + the whole cnn, ss_baselines/av_wan/models/map_cnn.py:65-104
 *   ssb_gru_step_batch      <- RNNStateEncoder.single_forward with a one-layer GRU under no_grad (rollout time),
 *                              ss_baselines/av_nav/models/rnn_state_encoder.py:80-90
 *   ssb_gru_seq_forward_batch / ssb_gru_seq_backward_batch <- RNNStateEncoder.seq_forward with a one-layer GRU and its
 *                              autograd backward (PPO's update), ss_baselines/av_nav/models/rnn_state_encoder.py:92-143
 *   ssb_policy_head_batch   <- Policy.act after self.net under no_grad (rollout time): the actor Linear of
 *                              CategoricalNet / CategoricalNetWithMask, CriticHead, CustomFixedCategorical's sample()
 *                              or mode() and log_probs(), ss_baselines/common/utils.py:41-87, av_nav/ppo/policy.py:
 *                              35-60, savi/ppo/policy.py:42-65, av_wan/ppo/policy.py:39-60
 *   ssb_policy_head_train_forward_batch / ssb_policy_head_train_backward_batch <- Policy.evaluate_actions after
 *                              self.net and its autograd backward (PPO's update): the same heads, log_probs() and
 *                              entropy(), av_nav/ppo/policy.py:70-82, savi/ppo/policy.py:73-93, av_wan/ppo/policy.py:68-80
 *   ssb_rollout_insert_batch / ssb_rollout_returns_batch / ssb_rollout_gather_batch <- RolloutStorage.insert
 *                              (with SAVi's ExternalMemory.insert), compute_returns (+ PPO.get_advantages),
 *                              recurrent_generator and after_update, ss_baselines/common/rollout_storage.py,
 *                              savi/models/rollout_storage.py
 *   ssb_belief_update_batch <- the per-env loops of BeliefPredictor.update after its two networks,
 *                              ss_baselines/savi/models/belief_predictor.py:150-175,181-202 with odom_to_base /
 *                              base_to_odom :210-226 (ppo_trainer.py:332-336, once per rollout step)
 *   ssb_resnet18_batch      <- BeliefPredictor's torchvision ResNet-18s under no_grad (rollout time): the label
 *                              classifier, belief_predictor.py:78-80,178-179, and the location predictor without
 *                              online training, :73-75,123-134,147-148
 *   ssb_smt_resnet18_batch  <- the location predictor with online training, custom_resnet18 of
 *                              ss_baselines/savi/models/smt_resnet.py, belief_predictor.py:66-71,123-134,147-148
 *   ssb_resnet18_train_forward_batch / _backward_batch <- AudioGoalPredictor.forward and its backward in SAVi's
 *                              pretraining, ss_baselines/savi/pretraining/audiogoal_predictor.py:29-38 as
 *                              audiogoal_trainer.py:69-124 trains it (BatchNorm in train() or eval())
 *   ssb_smt_cnn_batch       <- SMTCNN.forward under no_grad (rollout time), SAVi's visual encoder: permute, RGB / 255,
 *                              ResizeCenterCropper(64, 64) and one custom_resnet18 per modality,
 *                              ss_baselines/savi/models/smt_cnn.py:76-113, common/utils.py:341-466
 *   ssb_smt_state_encoder_batch <- SMTStateEncoder.single_forward under no_grad (rollout time), SAVi's scene memory
 *                              transformer, ss_baselines/savi/models/smt_state_encoder.py:92-245, called from
 *                              AudioNavSMTNet.forward, ss_baselines/savi/ppo/policy.py:380-403
 *   ssb_smt_state_encoder_train_forward_batch / _backward_batch <- SMTStateEncoder.single_forward under grad (PPO's
 *                              evaluate_actions), ss_baselines/savi/models/smt_state_encoder.py:92-157, and its backward
 *   ssb_map_update_batch    <- Mapper.reset / Mapper.update's map writes, ss_baselines/av_wan/models/mapper.py:77-137,
 *                              replayed from the records env workers send (soundspaces_b200.maps)
 *   ssb_map_observe_batch   <- Planner.add_maps_to_observation, av_wan/models/planner.py:76-83 (the three egocentric
 *                              crops of mapper.py:212-293)
 *   ssb_logmel_batch       <- EXTENSION (no reference code): the log-mel front end BASELINE.json configs[2] names;
 *                              log1p(librosa.feature.melspectrogram) on the reference's STFT geometry (nav.py:89-92)
 *   ssb_frame_gather_batch <- batch_obs's torch.stack([...]).float() of the rgb / depth observations,
 *                              ss_baselines/common/utils.py:126-153, for frames remote env workers send once
 *   ssb_pcm16_decode/encode <- int16 <-> float32 PCM (librosa.load decode used at
 *                              simulator.py:597; np.int16(audio*32767) at
 *                              scripts/interactive_demo.py:110)
 *
 * Conventions: every function returns 0 on success or a negative SSB_E* code and
 * never throws; ssb_last_error(ctx) describes the last failure.  All pointers
 * named d_* are device pointers on the context's device; h_* are host pointers
 * (pinned for asynchronous copies).  Work is enqueued on the caller's stream
 * (a cudaStream_t passed as void*; NULL = legacy default stream) and is
 * asynchronous; a context is not thread-safe.  No torch types cross this ABI.
 */
#ifndef SSB200_H
#define SSB200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SSB_OK 0
#define SSB_E_INVALID_ARG (-1)
#define SSB_E_CUDA (-2)
#define SSB_E_OOM (-3)
#define SSB_E_SHAPE (-4)

#define SSB_FLAG_SILENT 1u      /* simulator.py:610-612: exact zeros */

#define SSB_PAD_REFLECT 0       /* librosa < 0.10 default */
#define SSB_PAD_CONSTANT 1      /* librosa >= 0.10 default */
#define SSB_LAYOUT_NCHW 0x100   /* OR into pad_mode: emit (2, 65, T') per env instead of the reference's (65, T', 2) */

#define SSB_N_FFT 512           /* nav.py:89-91 */
#define SSB_HOP 160
#define SSB_WIN 400
#define SSB_POOL 4              /* nav.py:93 */
#define SSB_SPEC_ROWS 65        /* ceil(257 / 4) */

typedef struct ssb_ctx ssb_ctx;

/* One convolution term: out[m] += sum_{k < rir_taps} rir[k] * src_ext[m0 + m - k].
 * The source enters through its overlap-save window spectra (ssb_source_windows). */
typedef struct {
    int64_t rir_offset; /* first tap of the (taps, 2) float32 interleaved RIR, in taps from d_rir_bank */
    int64_t x_offset;   /* first element (float2 units) of the window spectra, from d_xpool */
    int32_t rir_taps;   /* taps to use = min(file taps, m0 + out_samples); 0 => term contributes nothing
                           (zero-RIR fallback simulator.py:617-624, or unused distractor slot) */
    int32_t x_nw;       /* number of windows stored at x_offset */
    int32_t x_wofs;     /* stored window j holds overlap-save block index j - x_wofs */
    int32_t reserved;
} ssb_conv_term;

typedef struct {
    ssb_conv_term term[2]; /* [0] the goal sound, [1] the distractor (simulator.py:649-664) */
    int32_t out_samples;   /* valid samples; [out_samples, sr) is zero (continuous_simulator.py:454) */
    uint32_t flags;        /* SSB_FLAG_* */
} ssb_req;

/* Two convolution plans:
 *  - partitioned overlap-save (log2n 12, 13 or 14): any RIR length, one or two terms; three kernels with the RIR
 *    spectra and the partition sums as L2-visible intermediates;
 *  - single block (log2n 16): ONE 65536-point circular convolution per env by a 4-CTA cluster, RIR FFT x source
 *    spectrum x inverse FFT fused in one kernel (no intermediate but the waveform); one term, RIRs of at most
 *    65536 - sr + 1 effective taps.  The source enters as ONE 65536-point spectrum per (clip, offset):
 *    ssb_source_windows with nw = 1, wofs = 0 writes 65536 float2; x_nw / x_wofs of the request are ignored. */
typedef struct {
    int32_t log2n;      /* 12, 13, 14: FFT size of the overlap-save blocks; 16: single-block plan */
    int32_t block;      /* P = 2^log2n / 2 output samples per block (log2n 16: the shift D = 65536 - sr) */
    int32_t sr;         /* samples per output row (RIR_SAMPLING_RATE) */
    int32_t n_blocks;   /* ceil(sr / P) (log2n 16: 1) */
    int32_t max_parts;  /* RIR partitions the scratch is sized for (log2n 16: 1) */
    int32_t n_terms;    /* 1 or 2 (log2n 16: 1) */
    int64_t h_elems_per_env; /* float2 elements of RIR-spectrum scratch per env (log2n 16: 0, d_hscratch unused) */
} ssb_plan;

int ssb_version(void);
int ssb_create(int device, ssb_ctx** out);
void ssb_destroy(ssb_ctx* ctx);
const char* ssb_last_error(const ssb_ctx* ctx);
/* kernels launched by this context since creation (for bench.py's gpu_launches) */
int64_t ssb_launch_count(const ssb_ctx* ctx);

/* Optional per-kernel timing for bench.py's roofline: when enabled every kernel launch is
 * bracketed by CUDA events on the launching stream.  ssb_get_kernel_timing synchronises, writes
 * the summed milliseconds and launch counts per kernel (index SSB_K_*) and clears the record. */
#define SSB_K_FWD_RIR 0
#define SSB_K_MAC_IFFT 1
#define SSB_K_SPECTROGRAM 2
#define SSB_K_FWD_SRC 3
#define SSB_K_MAC_BINS 4
#define SSB_K_CONV64K 5
#define SSB_N_KERNELS 6
int ssb_set_kernel_timing(ssb_ctx* ctx, int enable);
int ssb_get_kernel_timing(ssb_ctx* ctx, double* ms_sum /*[SSB_N_KERNELS]*/, int64_t* counts /*[SSB_N_KERNELS]*/);

/* Convolution schedule: 0 (default) = per-bin partition sums, then inverse FFTs: at log2n 12 in one cluster kernel
 * that passes the sums over distributed shared memory (timed as SSB_K_MAC_IFFT; SSB_K_MAC_BINS then counts 0
 * launches), at log2n 13 / 14 through an HBM intermediate (mac_bins_kernel, then mac_ifft_kernel);
 * 1 = partition sums fused into the inverse-FFT kernel (re-reads every RIR partition per block). */
int ssb_set_conv_mode(ssb_ctx* ctx, int mode);
/* ssb_render_batch splits the batch over n (1..8) internal streams forked from / joined to the
 * caller's stream, so kernel tails and memory- vs compute-bound kernels of different sub-batches overlap */
int ssb_set_streams(ssb_ctx* ctx, int n);

/* Each internal stream works through n sub-batches one after the other (default 1): sub-batches = streams x n,
 * at least 16 envs each.  Smaller sub-batches keep the per-step intermediates (partition spectra, partition sums,
 * waveform: 1.3 MB per env at 44.1 kHz / 16384 taps) inside the L2. */
int ssb_set_chunks(ssb_ctx* ctx, int n);

/* Test hook: flags = 32 forces the direct-form SH decode in ssb_sh_decode_batch (the reference the FFT form is
 * checked against), 0 restores the default.  Any other bit returns SSB_E_INVALID_ARG. */
int ssb_set_debug(ssb_ctx* ctx, int flags);

/* Fill a plan.  log2n = 0 picks the partitioned default (12; 13 when max_taps > 24576); log2n = 16 asks for the
 * single-block plan and fails with SSB_E_INVALID_ARG when n_terms != 1, sr > 61440 or max_taps > 65536 - sr + 1. */
int ssb_make_plan(ssb_ctx* ctx, int sr, int max_taps, int n_terms, int log2n, ssb_plan* plan);

/* spectrogram geometry: frames = 1 + sr/160, cols = ceil(frames/4) */
int ssb_spec_cols(int sr);

/* Overlap-save window spectra of one mono clip.  Window j (0 <= j < nw) covers source
 * samples [m0 + (j - wofs - 1) * P, m0 + (j - wofs + 1) * P); samples < 0 read as 0, samples >= S
 * read as src[n - S] when wrap != 0 (continuous_simulator.py:443-445) else 0.
 * d_x receives nw * 2^log2n float2. */
int ssb_source_windows(ssb_ctx* ctx, const ssb_plan* plan, const float* d_src, int S, int64_t m0, int wrap,
                       int nw, int wofs, void* d_x, void* stream);

/* Convolve a batch: d_wave[env][ear][n], row stride wave_stride floats (>= sr), ear 0 = left.
 * d_hscratch: B * plan->h_elems_per_env float2. */
int ssb_convolve_batch(ssb_ctx* ctx, const ssb_plan* plan, int B, const ssb_req* d_reqs,
                       const float* d_rir_bank, const void* d_xpool, void* d_hscratch,
                       float* d_wave, int64_t wave_stride, void* stream);

/* out[env][:, :n+1] = a*w1 + b*w2 over the first n+1 = int(0.05*sr)+1 samples, rest = b; in place on b. */
int ssb_crossfade_batch(ssb_ctx* ctx, int B, const float* d_prev, float* d_cur, int sr,
                        int64_t wave_stride, const uint8_t* d_enable, void* stream);

/* d_spec[env][65][cols][2] = log1p(mean4x4(|STFT(d_wave[env][ear])|)); d_spec must be 8-byte aligned unless
 * SSB_LAYOUT_NCHW is set (SSB_E_INVALID_ARG otherwise) */
int ssb_spectrogram_batch(ssb_ctx* ctx, int B, const float* d_wave, int64_t wave_stride, int sr,
                          int pad_mode, float* d_spec, void* stream);

/* convolve + spectrogram.  d_wave is required (it is the intermediate). */
int ssb_render_batch(ssb_ctx* ctx, const ssb_plan* plan, int B, const ssb_req* d_reqs,
                     const float* d_rir_bank, const void* d_xpool, void* d_hscratch,
                     float* d_wave, int64_t wave_stride, int pad_mode, float* d_spec, void* stream);

/* Host-buffer entry: copies h_rir (rir_bytes; offsets in h_reqs index it) and h_reqs to the device
 * staging buffers the caller provides, renders, and copies the spectrogram (and the waveform when
 * h_wave != NULL, densely packed [B][2][sr]) back to the host.  n_chunks > 1 splits the batch and
 * overlaps H2D copy / kernels / D2H copy of consecutive chunks on internal copy streams; either way
 * all of it is ordered after prior work on `stream` and `stream` completes when the results have
 * landed; the caller synchronises. */
int ssb_render_batch_host(ssb_ctx* ctx, const ssb_plan* plan, int B, const ssb_req* h_reqs,
                          const float* h_rir, int64_t rir_bytes, float* d_rir_staging, ssb_req* d_reqs_staging,
                          const void* d_xpool, void* d_hscratch, float* d_wave, int64_t wave_stride,
                          int pad_mode, float* d_spec, float* h_spec, float* h_wave, int n_chunks, void* stream);

/* bytes the last ssb_render_batch_host call copied host->device and device->host */
int ssb_host_copy_bytes(const ssb_ctx* ctx, int64_t* h2d, int64_t* d2h);

/* Ambisonic -> binaural decode of a batch of 9-channel (ACN, second order) impulse responses:
 * d_out_rir[env][n][ear] = sum_k sum_tau (R(az_env) a)_k[n - 128 - tau] * hbank[k][ear][tau], n < L,
 * i.e. what scripts/ambisonic_to_binaural.py:14-19 obtains from the closed AmbisonicBinauralizer
 * (rotation about the vertical axis, 9 x 2 FIR filters of 256 taps, 128-sample bulk delay, output
 * cut to the input length).  d_amb: [B][L][9] f32; d_az_deg: [B] f32 degrees; d_hbank: [9][2][256] f32;
 * d_filters: scratch of B * 9 * 256 float2; d_out_rir: [B][L][2] f32, directly usable as an RIR bank.
 * Azimuths: any finite value.  The kernel reduces it with fmodf(az, 360), which is exact, before converting to
 * radians, so az and az + 360 k decode alike and the accuracy does not depend on |az|.  The values are not inspected
 * on the host: a NaN or +-inf azimuth gives that env an all-NaN output and leaves the other envs' rows untouched.
 * B < 0, B > 65535, L <= 0, L > SSB_SH_MAX_L or a NULL or misaligned pointer (4 bytes for d_amb, d_az_deg and d_hbank,
 * 8 for d_filters and d_out_rir) returns SSB_E_INVALID_ARG before anything is launched; B = 0 does nothing. */
#define SSB_SH_MAX_L (1 << 30)  /* longest response either decode entry accepts, in samples */
int ssb_sh_decode_batch(ssb_ctx* ctx, int B, const float* d_amb, int L, const float* d_az_deg, const float* d_hbank,
                        void* d_filters, float* d_out_rir, void* stream);

/* The same decode at ambisonic orders 0 to 3 and several azimuths per input, reading each input once:
 * d_out[in][a][n][ear] = sum_k sum_tau (R(az_a) a_in)_k[n - 128 - tau] * hbank[k][ear][tau], n < L, with K = n_channels
 * in {1, 4, 9, 16} (ACN order; the third-order pairs (11,13), (10,14), (9,15) rotate by az, 2 az, 3 az).
 * d_amb: [n_inputs][L][K] f32; d_az_deg: [n_az] f32 degrees; d_hbank: [K][2][256] f32 (the first K rows of the 16-row
 * bank); d_filters: scratch of n_az * K * 256 float2; d_out: [n_inputs][n_az][L][2] f32.  A row is bit-identical to
 * the n_az = 1 decode at its azimuth, whatever n_inputs is and wherever the input sits in the batch.  Azimuths as for
 * ssb_sh_decode_batch: any finite value, reduced exactly; a NaN or +-inf azimuth gives all-NaN rows at that azimuth
 * only (at K = 1 nothing rotates and the azimuth is not used).  Another K, n_az < 1, n_inputs * n_az > 65535, L <= 0, L > SSB_SH_MAX_L or a NULL or misaligned pointer returns
 * SSB_E_INVALID_ARG before anything is launched; n_inputs = 0 does nothing. */
int ssb_sh_decode_multi_batch(ssb_ctx* ctx, int n_inputs, int n_channels, int L, const float* d_amb, int n_az,
                              const float* d_az_deg, const float* d_hbank, void* d_filters, float* d_out, void* stream);

/* AV-WaN Intensity sensor (ss_baselines/av_wan/avwan_sensors.py:91-100) for a batch of (2, sr)
 * waveforms: d_out[env] = mean(x[:, i:i+num_frame]**2), i = first sample (min over ears) above 10 % of
 * the clip maximum. */
int ssb_intensity_batch(ssb_ctx* ctx, int B, const float* d_wave, int64_t wave_stride, int sr, int num_frame,
                        float* d_out, void* stream);

/* EXTENSION -- the reference has no mel front end (SURVEY.md 8(d)); BASELINE.json configs[2] asks for one.
 * d_out[env][j][t][ear] = log1p(sum_k M[j][k] * |STFT(d_wave[env][ear])[k][t]|^power), power 1 or 2, t < 1 + sr/160,
 * STFT as in ssb_spectrogram_batch (n_fft 512, hop 160, Hann(400), centre padding per pad_mode), M the Slaney
 * filterbank of librosa.filters.mel(sr, 512, n_mels) with fmin 0, fmax sr/2 (n_mels <= 64), i.e.
 * log1p(librosa.feature.melspectrogram(y, sr, n_fft=512, hop_length=160, win_length=400, n_mels, power)).
 * ssb_mel_filterbank writes that matrix densely, [n_mels][257], to HOST memory (needs no device). */
int ssb_logmel_frames(int sr);
int ssb_mel_filterbank(int sr, int n_mels, float* h_out);
int ssb_logmel_batch(ssb_ctx* ctx, int B, const float* d_wave, int64_t wave_stride, int sr, int n_mels, int power,
                     int pad_mode, float* d_out, void* stream);

/* SURVEY.md N2: first layer of the policy's audio encoder, fused with the layout change.  AudioCNN.forward
 * (ss_baselines/av_nav/models/audio_cnn.py:79-89) permutes the observation to channels-first and applies
 * Conv2d(2 -> OC, KHxKW, stride SHxSW, no padding) [+ ReLU]; this reads d_spec[env][H][W][2] (the layout
 * ssb_spectrogram_batch writes) and writes d_out[env][OC][H1][W1], H1 = (H-KH)/SH + 1, W1 = (W-KW)/SW + 1.
 * d_weight: [OC][2][KH][KW] (torch's Conv2d.weight), d_bias: [OC] or NULL.  Inference only.  SSB_E_SHAPE when
 * W1 * OC > 1024 or the staged rows + weights exceed 48 KB. */
int ssb_audio_conv1_batch(ssb_ctx* ctx, int B, const float* d_spec, int H, int W, const float* d_weight,
                          const float* d_bias, int OC, int KH, int KW, int SH, int SW, int relu, float* d_out, void* stream);

/* One unpadded, undilated, ungrouped Conv2d of the audio encoder: d_weight [out_channels][in_channels][kh][kw] (torch's
 * Conv2d.weight; in_channels is 2 for the first layer and the previous layer's out_channels otherwise), d_bias
 * [out_channels] or NULL, stride sh x sw, relu 0 or 1. */
typedef struct {
    const float* d_weight;
    const float* d_bias;
    int32_t out_channels, kh, kw, sh, sw, relu;
} ssb_conv2d_layer;

/* The whole AudioCNN.cnn at rollout time (ss_baselines/{av_nav,av_wan,savi}/models/audio_cnn.py, forward = permute +
 * Conv2d ReLU Conv2d ReLU Conv2d Flatten Linear ReLU): reads d_spec[env][H][W][2] (the layout ssb_spectrogram_batch
 * writes), runs layers[0..2] (a host array), writes d_features[env][F] in torch's Flatten order (c, h, w),
 * F = C3 * H3 * W3, and d_out[env][j] = act(d_lin_bias[j] + sum_f d_lin_weight[j][f] * d_features[env][f]),
 * d_lin_weight [hidden][F], d_lin_bias [hidden] or NULL, act = ReLU when lin_relu = 1, identity when 0.  Every ReLU
 * keeps NaN, as torch's does, so NaN in an env's observation reaches its outputs as in the reference.  Inference
 * only, FP32.  An env's outputs are bit-identical whatever B and its position in the batch.
 * Limits, checked on the host before any launch (SSB_E_SHAPE with a message): every layer's output is non-empty, and
 * the observation, the conv1 and conv2 activations and the largest per-CTA weight slice,
 * H W 2 + C1 H1 W1 + C2 H2 W2 + max over layers of ceil(OC / 8) IC KH KW floats (each env runs on 8 CTAs, each
 * computing 1/8 of every layer's output channels), fit the kernel's 227 KB (232448 bytes) of shared memory.  There is
 * no per-layer thread limit (each CTA loops over its outputs).  SSB_E_INVALID_ARG: B < 0 or > 65535, H or W < 1,
 * hidden < 1, a relu flag not 0 / 1, a NULL d_spec, layer weight, d_lin_weight, d_features or d_out, or any pointer
 * (d_spec, a layer's d_weight or d_bias, d_lin_weight, d_lin_bias, d_features, d_out) not 4-byte aligned. */
int ssb_audio_encoder_batch(ssb_ctx* ctx, int B, const float* d_spec, int H, int W, const ssb_conv2d_layer layers[3],
                            const float* d_lin_weight, const float* d_lin_bias, int hidden, int lin_relu,
                            float* d_features, float* d_out, void* stream);

/* The same for SAVi with a distractor sound (ss_baselines/savi/models/audio_cnn.py:135-150): the network's input is
 * the observation with env n's category row d_labels[n][0..n_labels-1] (row stride label_stride floats) broadcast
 * over H x W and concatenated after the two ears, so layers[0].d_weight is [C1][2 + n_labels][KH][KW].  A label
 * channel is constant over the unpadded conv1's window, so it enters as the per-env bias
 * b[oc] + sum_c d_labels[n][c] * sum_{kh,kw} W[oc][2 + c][kh][kw], formed in the kernel in a fixed order.  NaN labels
 * give NaN as in torch, but the fold differs from torch's tap-by-tap sum for an infinite label: where a channel's taps
 * differ in sign, torch gives NaN and the fold gives +-Inf.  SAVi's category is one-hot or a probability, so infinite
 * labels are outside the supported domain.  The results are
 * bit-identical whatever B, the env's position and label_stride, and with n_labels = 0 (d_labels unused) bit-identical
 * to ssb_audio_encoder_batch.  Two launches, as there.  Shared memory as there with IC = 2 + n_labels for conv1:
 * H W 2 + C1 H1 W1 + C2 H2 W2 + max(ceil(C1 / 8) (2 + n_labels) KH1 KW1, ceil(C2 / 8) C1 KH2 KW2, ceil(C3 / 8) C2 KH3 KW3)
 * floats <= 232448 bytes, else SSB_E_SHAPE.  SSB_E_INVALID_ARG as there, and for n_labels < 0, n_labels > 0 with a NULL
 * or misaligned d_labels, and label_stride < n_labels.  All refusals are decided on the host before any launch. */
int ssb_audio_encoder_category_batch(ssb_ctx* ctx, int B, const float* d_spec, int H, int W,
                                     const ssb_conv2d_layer layers[3], const float* d_labels, int n_labels,
                                     int64_t label_stride, const float* d_lin_weight, const float* d_lin_bias,
                                     int hidden, int lin_relu, float* d_features, float* d_out, void* stream);

/* The whole VisualCNN.cnn at rollout time (ss_baselines/av_nav/models/visual_cnn.py:137-161, av_wan/models/
 * visual_cnn.py:95-118, savi/models/visual_cnn.py:163-188 without semantic channels; forward = permute + RGB / 255 +
 * cat + Conv2d ReLU Conv2d ReLU Conv2d Flatten Linear ReLU).  Reads d_rgb[env][H][W][n_rgb] and d_depth[env][H][W]
 * [n_depth] (the layout batch_obs delivers; a NULL pointer or a count of 0 means no such input), so layers[0].d_weight is
 * [C1][n_rgb + n_depth][KH][KW] with the RGB channels first.  Each RGB value is multiplied by the float32 1 / 255 as it is
 * loaded, which is what torch's CUDA x / 255.0 computes; the weights are used as given.  Writes d_features[env][F] in
 * torch's Flatten order (c, h, w), F = C3 H3 W3, and d_out[env][hidden] as ssb_audio_encoder_batch does; the ReLUs
 * keep NaN, so NaN or Inf in an env's observation gives that env's outputs float64's NaN / Inf pattern.  Two launches
 * per call, whatever B.  FP32 FMA, no tensor cores; every sum has an order fixed by the layer's shape, so an env's
 * outputs are bit-identical whatever B and its position in the batch.  Parameters are read through the pointers on
 * every call.  Each env runs on a cluster of 8 CTAs; conv1 is computed from the observation in global memory one
 * output row at a time.  Shared memory: C1 H1 W1 + max(C2 H2 W2, C1 IC KH1 KW1 + IC KH1 W) + max(ceil(C2 / 8) C1 KH2 KW2,
 * ceil(C3 / 8) C2 KH3 KW3) floats (IC = n_rgb + n_depth) must fit 232448 bytes: 191616 bytes for av_nav's RGB-D network
 * at 128 x 128.  SSB_E_INVALID_ARG: B < 0 or > 65535, n_rgb or n_depth < 0, no input channel, H or W < 1, a NULL or
 * misaligned pointer, hidden < 1, a relu flag not 0 / 1.  SSB_E_SHAPE, with the byte count in the message: a layer's
 * output is empty, or the shared memory above exceeds 232448 bytes (the 1024 x 1024 interactive_demo sensor); also
 * SSB_E_SHAPE, with the count in the message, for F > 2^31 - 1, which the shared-memory bound does not exclude (a
 * 120 x 120 input through 1 x 1 convs to 149131 channels fits it).  All decided on the host before any launch, whatever
 * B; B = 0 launches nothing. */
int ssb_visual_encoder_batch(ssb_ctx* ctx, int B, const float* d_rgb, int n_rgb, const float* d_depth, int n_depth,
                             int H, int W, const ssb_conv2d_layer layers[3], const float* d_lin_weight,
                             const float* d_lin_bias, int hidden, int lin_relu, float* d_features, float* d_out,
                             void* stream);

/* The whole MapCNN.cnn at rollout time, AV-WaN's geometric and acoustic map encoders
 * (ss_baselines/av_wan/models/map_cnn.py:65-104; forward = permute + Conv2d ReLU Conv2d ReLU Conv2d Flatten Linear ReLU,
 * unpadded, kernel sizes and strides per map type and size at :36-52).  Reads d_map[env][H][W][C] (observations["gm"] /
 * ["am"] as batch_obs delivers them), so layers[0].d_weight is [C1][C][KH][KW]; no scaling.  Writes d_features[env][F]
 * in torch's Flatten order (c, h, w), F = C3 H3 W3, and d_out[env][hidden] as ssb_audio_encoder_batch does; the ReLUs
 * keep NaN.  Two launches per call, whatever B.  FP32 FMA, no tensor cores; every sum is bias, then (ic, kh, kw) in
 * order, so an env's outputs are bit-identical whatever B and its position in the batch.  Parameters are read through
 * the pointers on every call.  Each env runs on a cluster of 8 CTAs with conv1's activations spread across it: rank r
 * keeps conv1 rows r, r + 8, ...; conv2 runs one output row at a time from the KH2 conv1 rows gathered over DSMEM,
 * each rank computing ceil(C2 / 8) channels; each rank then gathers the whole conv2 output and computes ceil(C3 / 8)
 * conv3 channels.  Shared memory per CTA, in floats:
 *   max(C1 ceil(H1 / 8) W1 + max(C1 C KH1 KW1 + C KH1 W, C1 KH2 W1 + ceil(C2 / 8) C1 KH2 KW2),
 *       C2 H2 W2 + ceil(C3 / 8) C2 KH3 KW3) + ceil(C2 / 8) H2 W2
 * must fit 232448 bytes: 161568 bytes for the 200 x 200 x 2 geometric map (MAP_SIZE 200), 169504 for 400 x 400 x 2
 * (MAP_SIZE 400), 19584 for the 20 x 20 x 1 acoustic map.  SSB_E_INVALID_ARG: B < 0 or > 65535, C, H or W < 1, hidden
 * < 1, a relu flag not 0 / 1, a NULL or misaligned pointer.  SSB_E_SHAPE, with the byte count in the message: a
 * layer's output is empty, or the shared memory above exceeds 232448 bytes; also SSB_E_SHAPE, with the count in the
 * message, for F > 2^31 - 1, which the shared-memory bound does not exclude (a 120 x 120 x 1 map through 1 x 1 convs to
 * 149131 channels fits it).  All decided on the host before any launch, whatever B; B = 0 launches nothing. */
int ssb_map_encoder_batch(ssb_ctx* ctx, int B, const float* d_map, int C, int H, int W,
                          const ssb_conv2d_layer layers[3], const float* d_lin_weight, const float* d_lin_bias,
                          int hidden, int lin_relu, float* d_features, float* d_out, void* stream);

/* One step of a one-layer nn.GRU with bias on masked state, RNNStateEncoder.single_forward
 * (ss_baselines/av_nav/models/rnn_state_encoder.py:80-90, also used by av_wan and SAVi's AudioNavBaselineNet):
 * h = d_masks[b] * d_h[b] (a multiply, so NaN in a done env's state propagates as in the reference), then
 * r = sigmoid(W_ir x + b_ir + W_hr h + b_hr), z = sigmoid(W_iz x + b_iz + W_hz h + b_hz),
 * n = tanh(W_in x + b_in + r (W_hn h + b_hn)), h' = (1 - z) n + z h, written to both d_out[b] and d_h_out[b].
 * d_x [B][I], d_h [B][Hd], d_masks [B], d_w_ih [3 Hd][I], d_w_hh [3 Hd][Hd], d_b_ih / d_b_hh [3 Hd] (torch's weight_ih_l0,
 * weight_hh_l0, bias_ih_l0, bias_hh_l0, rows in r, z, n order).  One launch; each weight row is read once per tile of
 * 16 envs.  FP32 FMA with full-precision expf / tanhf; every sum has an order fixed by I and Hd, so an env's outputs
 * are bit-identical whatever B and its position.  The host never reads the masks.  SSB_E_INVALID_ARG: B < 0 or
 * > 65535, I or Hd < 1, a NULL or misaligned pointer, d_out or d_h_out equal to d_h (no in-place update); decided on
 * the host before any launch; B = 0 launches nothing. */
int ssb_gru_step_batch(ssb_ctx* ctx, int B, int I, int Hd, const float* d_x, const float* d_h, const float* d_masks,
                       const float* d_w_ih, const float* d_w_hh, const float* d_b_ih, const float* d_b_hh, float* d_out,
                       float* d_h_out, void* stream);

/* RNNStateEncoder.seq_forward (ss_baselines/av_nav/models/rnn_state_encoder.py:92-143) with a one-layer nn.GRU with
 * bias, and its backward.  x [T N][I] (step-major, env-minor, as recurrent_generator lays out a minibatch), h0 [N][Hd],
 * masks [T N], parameters as ssb_gru_step_batch.  Step t of env e runs ssb_gru_step_batch's equations on h_prev =
 * masks[t N + e] * h_{t-1} when t is a segment start, and on h_prev = h_{t-1} (no multiply, whatever the mask)
 * otherwise; a segment start is t = 0 or a t >= 1 at which some env's mask equals 0.0, the steps at which the
 * reference splits the sequence.  The library decides them on the device; the host never reads the masks.
 *
 * Forward: d_out [T N][Hd] receives every step's state, d_h_last [N][Hd] the last one.  d_saved, when not NULL,
 * receives what the backward needs: 5 T N Hd floats, planes [T N][Hd] of h_prev, r, z, n and W_hn h_prev + b_hn.
 * Two launches: the input projection X W_ih^T + b_ih into the workspace, then the recurrence (a cooperative launch).
 *
 * Backward: from d_saved of a forward on the same x, masks and parameters, and the gradients of out and h_last
 * (either may be NULL: zero), writes d_dx [T N][I], d_dh0 [N][Hd] (through masks[0]), d_dw_ih [3 Hd][I],
 * d_dw_hh [3 Hd][Hd], d_db_ih and d_db_hh [3 Hd] (overwritten, not accumulated).  Any of the six may be NULL and is then
 * not computed; all six NULL launches nothing.  Launches: the reverse recurrence (cooperative), then one GEMM for d_dx,
 * one for d_dw_ih and / or d_db_ih, one for d_dw_hh and / or d_db_hh, each when requested.
 *
 * d_workspace: ssb_gru_seq_workspace_bytes(T, N, I, Hd) bytes, 16-byte aligned, for either entry; nothing in it
 * outlives a call.  FP32 FMA (no TF32) with full-precision expf / tanhf; every sum has an order fixed by the shapes and
 * there are no float atomics, so results are deterministic, and an env's out, h_last, dx and dh0 are bit-identical
 * whatever N and its position.  The launch count depends only on which gradients are requested.
 * Limits: 1 <= T <= SSB_GRU_SEQ_MAX_T, 1 <= N <= SSB_GRU_SEQ_MAX_N, 1 <= Hd <= SSB_GRU_SEQ_MAX_HD, I >= 1.
 * SSB_E_INVALID_ARG: a value outside the limits, a NULL or misaligned required pointer (all but d_saved in the
 * forward; d_x, d_masks, d_w_ih, d_w_hh, d_saved and d_workspace in the backward), a misaligned optional one, or an
 * output (out, h_last, saved, workspace; the gradients and workspace) overlapping an input or another output.
 * SSB_E_SHAPE: the device cannot hold the recurrence's grid at once (not on an H100).  Decided on the host before any
 * launch. */
#define SSB_GRU_SEQ_MAX_T 4096
#define SSB_GRU_SEQ_MAX_N 256
#define SSB_GRU_SEQ_MAX_HD 1024
int64_t ssb_gru_seq_workspace_bytes(int T, int N, int I, int Hd);  /* -1 outside the limits */
int ssb_gru_seq_forward_batch(ssb_ctx* ctx, int T, int N, int I, int Hd, const float* d_x, const float* d_h0,
                              const float* d_masks, const float* d_w_ih, const float* d_w_hh, const float* d_b_ih,
                              const float* d_b_hh, float* d_out, float* d_h_last, float* d_saved, void* d_workspace,
                              void* stream);
int ssb_gru_seq_backward_batch(ssb_ctx* ctx, int T, int N, int I, int Hd, const float* d_x, const float* d_masks,
                               const float* d_w_ih, const float* d_w_hh, const float* d_saved,
                               const float* d_grad_out, const float* d_grad_h_last, void* d_workspace, float* d_dx,
                               float* d_dh0, float* d_dw_ih, float* d_dw_hh, float* d_db_ih, float* d_db_hh,
                               void* stream);

/* The CNN encoders' conv stack for PPO's update: AudioCNN (all three baselines; SAVi's goal_encoder too), VisualCNN
 * (av_nav, savi's rnn policy) and AV-WaN's MapCNN, i.e. Conv2d ReLU Conv2d ReLU Conv2d Flatten Linear ReLU, unpadded,
 * forward and backward.  The input is one of three kinds, as the inference entries read them:
 *   SSB_CONV_INPUT_SPECTROGRAM  d_x [B][H][W][2] (channels = 2), optionally with SAVi's category rows
 *                               d_labels[n][0..n_labels-1] (row stride label_stride floats) as conv1 input channels
 *                               2..n_labels+1, folded into a per-env conv1 bias as ssb_audio_encoder_category_batch does;
 *   SSB_CONV_INPUT_VISUAL       RGB d_x [B][H][W][channels] times float32(1/255), then depth d_depth [B][H][W][n_depth]
 *                               (a NULL pointer or a count of 0 means no such input), as ssb_visual_encoder_batch;
 *   SSB_CONV_INPUT_MAP          d_x [B][H][W][channels], as ssb_map_encoder_batch.
 * layers[3] as ssb_audio_encoder_batch (conv1's d_weight [C1][IC + n_labels][KH][KW]), then the Linear: d_lin_weight
 * [hidden][lin_in_features], which must equal conv3's C3 H3 W3, d_lin_bias [hidden] or NULL, lin_relu 0 or 1.
 *
 * Forward: writes d_features [B][F] (conv3's output in Flatten order) and d_out [B][hidden], bit-identical to the
 * inference entry of the same input at any B and env position, and keeps conv1's and conv2's outputs in d_workspace
 * (ssb_conv_stack_train_workspace_bytes(..., backward = 0) bytes, 16-byte aligned), which the backward reads as
 * d_saved.  Launches: one per conv, one for the Linear (audio_encoder_linear_kernel), one more with labels: 4 or 5.
 *
 * Backward: from d_saved, d_features and d_out of a forward on the same input and parameters and the gradient of out,
 * overwrites the requested gradients: d_grad_weight[i] / d_grad_bias[i] for conv i (i < 3) and the Linear (i = 3),
 * each NULL when not wanted (the observation and the labels get none).  d_workspace: ...(backward = 1) bytes, 16-byte
 * aligned.  Order: the Linear's ReLU mask, dW / db of the Linear (one GEMM), dF = g W_lin, then from conv3 down to the
 * lowest conv with a requested gradient: dW / db (a GEMM in chunks of 2048 (env, pixel) rows, then the chunks summed in
 * order) and, below the top conv, dX by a gather-form transposed conv.  The ReLU masks follow torch's
 * threshold_backward (the gradient passes where !(output <= 0), so NaN passes).  A label channel's tap gradients are
 * all sum_n labels[n][c] sum_pos g1[n][oc][pos] (two launches).  Launches with every gradient requested: 11, 13 with
 * labels; fewer when the lower convs need nothing.  No float atomics: results are deterministic, and an env's dX does
 * not depend on B or its position.
 *
 * Every product is an FP32 fmaf (no TF32, no tensor cores).  Limits, checked on the host before any launch: B <=
 * SSB_CONV_STACK_MAX_B; n_labels <= SSB_CONV_STACK_MAX_LABELS; per layer IC KH KW and OC ceil(KH / SH) ceil(KW / SW)
 * (conv2, conv3) at most SSB_CONV_STACK_MAX_K; B H W, every layer's B C H W and B hidden at most 2^31 - 1; conv2's
 * and conv3's SH SW at most SSB_CONV_STACK_MAX_STRIDE_AREA (dX runs one grid z-slice per residue class
 * (ih mod SH, iw mod SW)); hidden at most SSB_CONV_STACK_MAX_HIDDEN (the Linear's dW runs 64 rows of it per grid y
 * index).  B and n_labels past their limits are SSB_E_INVALID_ARG; the other limits are SSB_E_SHAPE, as are an empty
 * layer output and lin_in_features != C3 H3 W3.  SSB_E_INVALID_ARG also: an unknown kind, a NULL or misaligned
 * pointer, a relu flag not 0 / 1, or an output (features, out, workspace; the gradients and the workspace)
 * overlapping an input or another output.  B = 0 launches nothing.
 * Kernels (-Xptxas -v, sm_90a): cs_gemm_kernel in its five instances 77-80 registers, no spills, 10752 B static shared
 * memory + 16 K B dynamic (K = the layer's GEMM columns); cs_reduce_kernel 32, cs_relu_grad_kernel 10,
 * cs_label_bias / sum / grad_kernel 30 / 32 / 32 registers, no spills. */
#define SSB_CONV_INPUT_SPECTROGRAM 0
#define SSB_CONV_INPUT_VISUAL 1
#define SSB_CONV_INPUT_MAP 2
#define SSB_CONV_STACK_MAX_B 65535
#define SSB_CONV_STACK_MAX_K 2048
#define SSB_CONV_STACK_MAX_LABELS 256
#define SSB_CONV_STACK_MAX_STRIDE_AREA 65535
#define SSB_CONV_STACK_MAX_HIDDEN 4194240
typedef struct {
    const float* d_x;
    const float* d_depth;
    const float* d_labels;
    int64_t label_stride;
    int32_t kind, H, W, channels, n_depth, n_labels;
} ssb_conv_stack_input;
int64_t ssb_conv_stack_train_workspace_bytes(int B, const ssb_conv_stack_input* in, const ssb_conv2d_layer layers[3],
                                             int lin_in_features, int hidden, int backward);  /* -1 when refused */
int ssb_conv_stack_train_forward_batch(ssb_ctx* ctx, int B, const ssb_conv_stack_input* in,
                                       const ssb_conv2d_layer layers[3], const float* d_lin_weight,
                                       const float* d_lin_bias, int lin_in_features, int hidden, int lin_relu,
                                       float* d_features, float* d_out, void* d_workspace, void* stream);
int ssb_conv_stack_train_backward_batch(ssb_ctx* ctx, int B, const ssb_conv_stack_input* in,
                                        const ssb_conv2d_layer layers[3], const float* d_lin_weight,
                                        int lin_in_features, int hidden, int lin_relu, const float* d_features,
                                        const float* d_out, const void* d_saved, const float* d_grad_out,
                                        void* d_workspace, float* const d_grad_weight[4], float* const d_grad_bias[4],
                                        void* stream);

/* The policy's action and value heads, Policy.act after self.net (ss_baselines/av_nav/ppo/policy.py:35-60,
 * savi/ppo/policy.py:42-65, av_wan/ppo/policy.py:39-60), for envs 0..B-1 in one launch.  d_features [B][H];
 * d_actor_weight [A][H] / d_actor_bias [A] (action_distribution.linear); d_critic_weight [H] / d_critic_bias [1]
 * (critic.fc).  value[b] = Wc f + bc; z = Wa f + ba.
 *  - masked = 0, CategoricalNet (common/utils.py:58-69): logits l = z - logsumexp(z), probs p = softmax(l),
 *    log_prob = l[action].  d_mask must be NULL.
 *  - masked = 1, CategoricalNetWithMask (:72-87): p = softmax(z), times d_mask [B][A] as a value when it is not NULL
 *    (masking on), then p / sum(p) (the probs of Categorical(probs=...)); log_prob = log(clamp(p[action], FLT_EPSILON,
 *    1 - FLT_EPSILON)), torch's probs_to_logits gathered without renormalising.
 * action = argmax(p / q) with d_q [B][A] the Exp(1) draws torch.multinomial(p, 1, True) makes (ATen's single-sample
 * path, the same generator call gives the same action), or argmax(p) when d_q is NULL (mode()); ties and NaN follow
 * torch.argmax (NaN first, then the lowest index).  d_probs [B][A], optional, receives p.  A row is refused where the
 * reference's validated constructor or multinomial raises: with masked = 0 a NaN in z - logsumexp(z), that is a NaN z,
 * any +Inf z or every z -Inf (some -Inf z beside finite ones are accepted, with probability 0); with masked = 1 a zero
 * sum, a NaN or a negative entry after normalising; with d_q, a non-finite p.  The reference's simplex tolerance
 * (|sum(p) - 1| < 1e-6) is not restated.  A refused row gets action -1 and NaN value, log_prob and probs;
 * *d_status receives the number of refused rows.  FP32 with FMA, full-precision expf / logf; every sum has an order
 * fixed by H and A, so an env's outputs are bit-identical whatever B and its position.  The count goes through a
 * context-owned ticket, so calls on one context must not overlap in time on different streams.
 * SSB_E_INVALID_ARG: B < 0 or > 65535, H or A < 1, masked not 0 / 1, d_mask with masked = 0, a NULL required pointer
 * (all but d_mask, d_q, d_probs) or a misaligned pointer (d_action: 8 bytes, the rest 4).  SSB_E_SHAPE: A > 256 or
 * H > 2048.  Decided on the host before any launch; B = 0 launches nothing and writes nothing, *d_status included. */
int ssb_policy_head_batch(ssb_ctx* ctx, int B, int H, int A, const float* d_features, const float* d_actor_weight,
                          const float* d_actor_bias, const float* d_critic_weight, const float* d_critic_bias,
                          int masked, const float* d_mask, const float* d_q, float* d_value, int64_t* d_action,
                          float* d_log_prob, float* d_probs, int* d_status, void* stream);

/* The same heads in PPO's update: Policy.evaluate_actions after self.net (ss_baselines/av_nav/ppo/policy.py:70-82,
 * savi/ppo/policy.py:73-93, av_wan/ppo/policy.py:68-80) for given actions, and torch's autograd of it.  Arguments
 * as ssb_policy_head_batch; d_action [B] int64 is an input.
 *
 * Forward, one launch: d_value [B] and d_log_prob [B] as ssb_policy_head_batch computes them (the same device code,
 * so for the same features, weights and action they are bit-identical to what it returned in the mode path);
 * d_entropy [B] the per-row entropy() of torch, -(clamp(logits, finfo.min) * probs).sum(-1), with logits the
 * log-probabilities (masked = 0) or log(clamp(p, FLT_EPSILON, 1 - FLT_EPSILON)) (masked = 1); d_saved [B][A] what the
 * backward reads: the log-probabilities (masked = 0) or softmax(z) before the mask (masked = 1).  A row is refused
 * where ssb_policy_head_batch refuses it without d_q, or where its action is outside [0, A) (log_prob's
 * _validate_sample); it gets NaN value, log_prob and entropy, and *d_status receives the number of refused rows,
 * through the context's ticket as in ssb_policy_head_batch.
 *
 * Backward, at most two launches: from d_saved of a forward on the same inputs and the gradients of value, log_prob
 * and entropy ([B] each), writes d_dfeatures [B][H], d_dactor_weight [A][H], d_dactor_bias [A], d_dcritic_weight [H]
 * and d_dcritic_bias [1] (overwritten); any may be NULL and is then not computed, all NULL launches nothing.  Launch
 * one gives dfeatures and the gradient of the actor's outputs, launch two (only when a parameter gradient is asked
 * for) the parameter gradients.  The clamps follow torch: clamp_probs passes gradient only where FLT_EPSILON <= p <=
 * 1 - FLT_EPSILON, the entropy's finfo.min clamp only where logits >= finfo.min, so rows with some -Inf logits get
 * finite gradients.  A row's dfeatures does not depend on B or its position; parameter gradients sum rows in an
 * order fixed by B, with no float atomics, so every result is bit-identical from run to run.
 *
 * d_workspace: ssb_policy_head_train_workspace_bytes(B, H, A) bytes, 16-byte aligned, for the backward; nothing in
 * it outlives a call.  Limits: 0 <= B <= SSB_POLICY_HEAD_TRAIN_MAX_B, the largest minibatch of the patched
 * recurrent_generator (soundspaces_b200/rollout.py).  SSB_E_INVALID_ARG: B outside the limit, H or A < 1, masked not
 * 0 / 1, d_mask with masked = 0, a NULL required pointer (every one but d_mask; in the backward also but the five
 * gradients) or a misaligned pointer (d_action 8 bytes, d_workspace 16, the rest 4).  SSB_E_SHAPE: A > 256 or
 * H > 2048.  Decided on the host before any launch; B = 0 launches nothing and writes nothing. */
#define SSB_POLICY_HEAD_TRAIN_MAX_B (4096 * 256)
int64_t ssb_policy_head_train_workspace_bytes(int B, int H, int A);  /* -1 outside the limits */
int ssb_policy_head_train_forward_batch(ssb_ctx* ctx, int B, int H, int A, const float* d_features,
                                        const float* d_actor_weight, const float* d_actor_bias,
                                        const float* d_critic_weight, const float* d_critic_bias, int masked,
                                        const float* d_mask, const int64_t* d_action, float* d_value,
                                        float* d_log_prob, float* d_entropy, float* d_saved, int* d_status,
                                        void* stream);
int ssb_policy_head_train_backward_batch(ssb_ctx* ctx, int B, int H, int A, const float* d_features,
                                         const float* d_actor_weight, const float* d_critic_weight, int masked,
                                         const float* d_mask, const int64_t* d_action, const float* d_saved,
                                         const float* d_grad_value, const float* d_grad_log_prob,
                                         const float* d_grad_entropy, void* d_workspace, float* d_dfeatures,
                                         float* d_dactor_weight, float* d_dactor_bias, float* d_dcritic_weight,
                                         float* d_dcritic_bias, void* stream);

/* PPO's rollout storage on the device (ss_baselines/common/rollout_storage.py, savi/models/rollout_storage.py,
 * soundspaces_b200/rollout.py).  The copies of all three entries are described by fields: row r = (o, t, j) of a
 * field is row_bytes bytes read from src + o * src_outer_stride + t * src_t_stride + col(j) * row_bytes and written to
 * dst + ((o * T + t) * n_cols + j) * row_bytes, with col(j) = h_cols[j] where the entry takes columns and j
 * otherwise.  Bytes are copied as they are, whatever the element type.  Limits of every field: T and outer >= 1,
 * row_bytes >= 1, outer * T * n_cols * row_bytes < 2^46, non-negative strides. */
#define SSB_ROLLOUT_MAX_FIELDS 32
#define SSB_ROLLOUT_MAX_COLS 256
#define SSB_ROLLOUT_MAX_ENVS 65535
#define SSB_ROLLOUT_MAX_STEPS 4096
#define SSB_ROLLOUT_MAX_MEMORY 16384
typedef struct {
    const void* src;
    void* dst;
    int64_t row_bytes;
    int64_t src_t_stride;
    int64_t src_outer_stride;   /* 0 repeats the source outer times */
    int32_t T;
    int32_t outer;
    int32_t on_host;            /* 1: src is host memory (ssb_rollout_insert_batch only; T = 1, one block) */
    int32_t reserved;
} ssb_rollout_field;

/* SAVi's ExternalMemory (savi/models/rollout_storage.py:347-377): d_masks [N][total], d_status [1 + N] int32. */
typedef struct {
    float* d_masks;
    const float* not_done;      /* [N] the step's not_done_masks, on the device or (not_done_on_host) the host */
    float* d_em_masks_out;      /* [N][total] (em_masks[step + 1]) or NULL */
    int* d_status;
    int32_t total, capacity, idx, step;
    int32_t not_done_on_host, reserved;
} ssb_rollout_memory;

/* RolloutStorage.insert (common :78-103, savi :103-130) in ONE launch: every field (T = 1 and n_cols = 1, so a field
 * is outer copies of one row_bytes block: the sensors, the hidden state, actions into actions[step] and
 * prev_actions[step + 1], log-prob, value, reward, mask; with a memory, the features into every copy of memory[idx]).
 * Fields with on_host (and a not_done_on_host) are copied by the host into one of a ring of 4 pinned,
 * device-mapped buffers, which the kernel reads, so nothing waits for the device unless that slot is still being
 * read by the launch 4 calls back.  With em (not NULL), per env row e of
 * d_masks in the reference's order: s = the row's sum (fixed order; equal to the reference's sum whenever the partial
 * sums are exact, as for 0 / 1 masks), s > capacity counts into d_status[0] and sets d_status[1 + e] to step + 1 if it
 * is 0; s == capacity clears column (idx - capacity) mod total; column idx is set to 1; the row is multiplied by
 * not_done[e] and written to d_em_masks_out when given.  SSB_E_INVALID_ARG: N < 1, n_fields < 0 or > 32, a NULL
 * pointer a field or the memory needs, a misaligned float pointer, on_host not 0 / 1, a host field with T != 1 or a
 * non-zero outer stride, idx outside [0, total), capacity outside [0, total].
 * SSB_E_SHAPE: N > 65535, total > 16384, a field beyond the limits above.  Decided before anything is staged. */
int ssb_rollout_insert_batch(ssb_ctx* ctx, int N, const ssb_rollout_field* fields, int n_fields,
                             const ssb_rollout_memory* em, void* stream);

/* RolloutStorage.compute_returns (common :105-129, savi :149-167) and PPO.get_advantages (av_nav/ppo/ppo.py:
 * 53-58, savi/ppo/ppo.py:54-59) for N envs in ONE launch of one CTA.  Tensors are [rows][N] float32: d_rewards
 * [S], d_value_preds / d_returns / d_masks [S + 1].  With scan = 1, over t = T-1 .. 0 (T <= S) and in float32 with
 * every operation rounded once, as the eager ops are: with use_gae, value_preds[T] = next_value, delta = (r[t] +
 * (gamma * v[t+1]) * m[t+1]) - v[t], gae = delta + (gamma_tau * m[t+1]) * gae, returns[t] = gae + v[t]; without,
 * returns[T] = next_value, returns[t] = (returns[t+1] * gamma) * m[t+1] + r[t].  gamma and gamma_tau are the float32
 * roundings of the Python floats gamma and gamma * tau.  With d_adv, then adv = returns[:S] - value_preds[:S], and with
 * normalize (x - mean) / (std + 1e-5): mean and the unbiased std summed in float64 in an order fixed by S and N,
 * rounded to float32 like torch's scalars, the last two operations in float32.  SSB_E_INVALID_ARG: N < 1, S < 1, T
 * outside [0, S], flags not 0 / 1, a NULL or misaligned pointer the call needs, scan = 0 without d_adv.  SSB_E_SHAPE:
 * N > 65535, S > 4096. */
int ssb_rollout_returns_batch(ssb_ctx* ctx, int N, int S, int T, int scan, int use_gae, float gamma, float gamma_tau,
                              const float* d_rewards, float* d_value_preds, float* d_returns, const float* d_masks,
                              const float* d_next_value, float* d_adv, int normalize, void* stream);

/* RolloutStorage.recurrent_generator's stacks for one minibatch (common :131-211, savi :169-292) and
 * RolloutStorage.after_update's copies into slot 0, in ONE launch: every field as above with n_cols columns, taken
 * from h_cols (host int64 [n_cols], each in [0, max_col)) or, with h_cols NULL, columns 0 .. n_cols-1.
 * SSB_E_INVALID_ARG: n_fields < 1 or > 32, n_cols < 1, a NULL field pointer, a host field, a column outside
 * [0, max_col).
 * SSB_E_SHAPE: n_cols > 256 with h_cols, n_cols > 65535, a field beyond the limits above. */
int ssb_rollout_gather_batch(ssb_ctx* ctx, const ssb_rollout_field* fields, int n_fields, int n_cols,
                             const int64_t* h_cols, int64_t max_col, void* stream);

/* SAVi's belief update (BeliefPredictor.update, ss_baselines/savi/models/belief_predictor.py:136-202) after the
 * location predictor and the label classifier have run, for envs 0..B-1 in one launch.  Env i is silent when every
 * element of d_spec[i] (H x W x 2 floats) is 0.  For the spectrogram (>= 0; NaN and Inf count as sounding) that is the
 * reference's sum() == 0; the two differ only for finite values of both signs that cancel to exactly 0.
 *  - location (d_loc_pred != NULL; [B][loc_stride], columns 0 and 1): reset the env's state when h_dones[i];
 *    sounding: base = (-p[1], p[0]); avg = base without a state or with current_pred_only, else
 *    (1-w) base + w odom_to_base(state, pose); state = base_to_odom(avg, pose).  Silent: avg = (10, 10) without a
 *    state, else odom_to_base(state, pose).  d_loc_out[i][0..1] = avg.  d_pose: [B][pose_stride], x, y, heading.
 *  - label (d_label_pred != NULL; [B][label_stride], columns 0..20): reset when h_dones[i]; sounding: avg = label
 *    without a state or with current_pred_only, else (1-w) label + w state; state = avg.  Silent: avg = 1/21
 *    without a state, else state.  d_cat_out[i][0..20] = avg.
 * State, kept by the caller across calls: d_last_pg [num_env][2], d_loc_valid [num_env], d_last_label [num_env][21],
 * d_label_valid [num_env] (0: no state; zero them to start); rows >= B are not touched.  h_dones: B host bytes
 * (non-zero = done) or NULL, packed into the launch's parameters (no copy).  Float32 in the reference's numpy order:
 * float32(1 - w) and float32(w), each product and sum rounded on its own, correctly rounded sqrt, full-precision
 * sin / cos / atan2.  The label belief is bit-identical to the reference's; the location belief differs by the ulp
 * errors of sin, cos and atan2.  SSB_E_INVALID_ARG: B > num_env, a NULL or misaligned pointer a requested belief
 * needs, loc_stride < 2, pose_stride < 3, label_stride < 21, current_pred_only not 0 / 1; SSB_E_SHAPE: B > 1024.
 * Both decided on the host before any launch.  With both predictions NULL nothing is launched. */
int ssb_belief_update_batch(ssb_ctx* ctx, int B, int num_env, const float* d_spec, int H, int W, const float* d_pose,
                            int64_t pose_stride, const float* d_loc_pred, int64_t loc_stride, const float* d_label_pred,
                            int64_t label_stride, const uint8_t* h_dones, double w, int current_pred_only,
                            float* d_last_pg, uint8_t* d_loc_valid, float* d_last_label, uint8_t* d_label_valid,
                            float* d_loc_out, float* d_cat_out, void* stream);

/* One convolution of a belief-predictor ResNet-18 with the norm that follows it.  d_weight: [OC][IC][KH][KW] (torch's
 * Conv2d.weight, bias-free); d_gamma / d_beta: [OC], the norm's weight and bias; d_mean / d_var: [OC], BatchNorm's
 * running statistics (ssb_resnet18_batch; unused by ssb_smt_resnet18_batch); eps > 0.  Parameters are read on every
 * call, so an optimiser step or a changed running statistic takes effect on the next call. */
typedef struct {
    const float* d_weight;
    const float* d_gamma;
    const float* d_beta;
    const float* d_mean;
    const float* d_var;
    float eps;
    int32_t reserved;
} ssb_resnet_conv;

/* SAVi's label classifier (and its location predictor without online training) at rollout time: torchvision's
 * resnet18 with conv1 = Conv2d(2, 64, 7, 2, 3, bias=False) and fc = Linear(fc_in = 512, n_out), BatchNorm in eval mode,
 * ss_baselines/savi/models/belief_predictor.py:73-80 as called by BeliefPredictor.update at :147-148 (cnn_forward
 * :123-134) and :178-179.  Reads d_spec[env][H][W][2] (the layout ssb_spectrogram_batch writes; the permute is folded
 * into the first conv's loads) and writes d_out[env][n_out] (d_fc_bias [n_out] or NULL).  convs: a host array of 20
 * in the module order conv1/bn1, then for each of layer1..layer4 and each of its two blocks: conv1/bn1, conv2/bn2 and,
 * in the first block of layer2..layer4, downsample.0/downsample.1.  Every layer runs from the live parameters: BatchNorm
 * is (x - running_mean) gamma / sqrt(running_var + eps) + beta, computed in the kernel on every call.  FP32 throughout,
 * no tensor cores; an env's outputs are bit-identical whatever B and its position (every sum has an order fixed by the
 * layer's shape).  39 launches per call, whatever B.  SSB_E_INVALID_ARG: B < 0, H or W < 1, n_out < 1, a NULL or
 * misaligned pointer, eps <= 0.  SSB_E_SHAPE: B > 1024, H or W > 256, fc_in != 512.  Both decided on the host before
 * any launch; B = 0 launches nothing. */
int ssb_resnet18_batch(ssb_ctx* ctx, int B, const float* d_spec, int H, int W, const ssb_resnet_conv convs[20],
                       const float* d_fc_weight, const float* d_fc_bias, int fc_in, int n_out, float* d_out, void* stream);

/* SAVi's location predictor with online training: custom_resnet18 of ss_baselines/savi/models/smt_resnet.py with
 * fc = Linear(fc_in, n_out), belief_predictor.py:66-71, as called through cnn_forward (:123-134) at :147-148.  Stem
 * Conv2d(2 + n_labels, 16, 7, 1, 3) + GroupNorm(16, 16) + ReLU; four stages of two BasicBlocks at widths 16/32/64/128
 * (3x3 convs, stride 2 and a 1x1 stride-2 conv + GroupNorm downsample in the first block of stages 2-4), every norm
 * GroupNorm(16, C): biased variance over (C/16 channels x H x W) per env and group, reduced in a fixed order; no
 * pooling, flatten in (c, h, w) order, so fc_in must be 128 H4 W4 (4608 for the 65 x 26 observation).  Input channel
 * 2 + c is env n's category d_labels[n][c] (row stride label_stride floats) where a tap lands inside the image and 0 in
 * the padding (cnn_forward's expand + cat, :126-129).  convs as in ssb_resnet18_batch with d_mean / d_var unused.
 * 38 launches per call, whatever B.  Numerics and refusals as ssb_resnet18_batch, plus SSB_E_INVALID_ARG for
 * n_labels < 0, n_labels > 0 with a NULL or misaligned d_labels, label_stride < n_labels, and SSB_E_SHAPE for
 * fc_in != 128 H4 W4. */
int ssb_smt_resnet18_batch(ssb_ctx* ctx, int B, const float* d_spec, int H, int W, const float* d_labels, int n_labels,
                           int64_t label_stride, const ssb_resnet_conv convs[20], const float* d_fc_weight,
                           const float* d_fc_bias, int fc_in, int n_out, float* d_out, void* stream);

/* The location predictor of ssb_smt_resnet18_batch for online training (ss_baselines/savi/ppo/ppo_trainer.py:342-400,
 * train_belief_predictor): a forward that keeps what the backward needs, and the backward of the parameters.
 *
 * ssb_smt_resnet18_train_workspace_bytes: bytes of the one workspace both entries use (16-byte aligned), or -1 when
 * the shape is refused.  It holds the forward's saved tensors (every conv's pre-norm sums, the GroupNorm statistics,
 * the stem, conv1 and block outputs) and the backward's scratch; the forward writes it, the backward reads it and
 * overwrites its scratch part, so a backward needs the workspace of its own forward, untouched in between.
 *
 * ssb_smt_resnet18_train_forward_batch: arguments and d_out as ssb_smt_resnet18_batch, with B <= 65535 instead of
 * 1024.  It runs the inference entry's conv, finish and head kernels with the same K splits, so d_out is
 * bit-identical to ssb_smt_resnet18_batch's for every row at any B and row order.  38 launches, whatever B.
 *
 * ssb_smt_resnet18_train_backward_batch: from d_dpred [B][n_out], the gradient of d_out, and the workspace of the
 * forward with the same arguments, writes the gradients of the 20 conv weights, the 20 GroupNorm gamma and beta, and
 * fc's weight and bias; any of them may be NULL (not computed).  The input and the labels get no gradient.  A row whose
 * d_dpred row is all zero contributes nothing and costs nothing: the first launch lists the other rows on the device
 * (a row holding NaN stays in the list), every later kernel reads that count from device memory, and every sum over
 * rows runs in list order, so the gradients are bit-identical to those of the same call without the silent rows.
 * FP32 FMA, no TF32 and no float atomics: two runs give the same bits.  With every gradient requested: 80 launches,
 * 82 with labels, whatever B and the number of live rows.
 *
 * Both: SSB_E_INVALID_ARG for what ssb_smt_resnet18_batch refuses, a NULL or misaligned workspace, and output buffers
 * (d_out, the workspace, the gradients) that overlap each other or an input; SSB_E_SHAPE for B > 65535, H or W > 256,
 * fc_in != 128 H4 W4.  Decided on the host before any launch; B = 0 launches nothing. */
int64_t ssb_smt_resnet18_train_workspace_bytes(int B, int H, int W, int n_labels, int n_out);
int ssb_smt_resnet18_train_forward_batch(ssb_ctx* ctx, int B, const float* d_spec, int H, int W, const float* d_labels,
                                         int n_labels, int64_t label_stride, const ssb_resnet_conv convs[20],
                                         const float* d_fc_weight, const float* d_fc_bias, int fc_in, int n_out,
                                         float* d_out, void* d_workspace, void* stream);
int ssb_smt_resnet18_train_backward_batch(ssb_ctx* ctx, int B, const float* d_spec, int H, int W, const float* d_labels,
                                          int n_labels, int64_t label_stride, const ssb_resnet_conv convs[20],
                                          const float* d_fc_weight, int fc_in, int n_out, const float* d_dpred,
                                          void* d_workspace, float* const d_dweight[20], float* const d_dgamma[20],
                                          float* const d_dbeta[20], float* d_dfc_weight, float* d_dfc_bias,
                                          void* stream);

/* SAVi's audio-goal predictor trained (ss_baselines/savi/pretraining/audiogoal_trainer.py:69-124, AudioGoalPredictor
 * of audiogoal_predictor.py:18-38): the network of ssb_resnet18_batch, with BatchNorm in training or eval mode, as a
 * forward that keeps what the backward needs and the backward of the parameters.
 *
 * ssb_resnet18_train_workspace_bytes: bytes of the one workspace both entries use (16-byte aligned), or -1 when the
 * shape is refused.  It holds the forward's saved tensors (every conv's pre-norm sums, the batch statistics, the
 * stem, conv1 and block outputs, the maxpool output and its window indices) and the backward's scratch; the forward
 * writes it, the backward reads it and overwrites its scratch part, so a backward needs the workspace of its own
 * forward, untouched in between.
 *
 * ssb_resnet18_train_forward_batch: arguments and d_out as ssb_resnet18_batch, with B <= 65535 instead of 1024.
 * bn_training = 1 is nn.BatchNorm2d.forward in train(): every norm normalises with its batch mean and biased variance
 * over (B, H, W) per channel, summed in FP64 in a fixed order, and updates d_mean / d_var in place to (1 - momentum)
 * r + momentum stat, with the unbiased variance (N / (N - 1)) for d_var, and adds 1 to each non-NULL
 * d_num_batches_tracked[i] (torch's int64 counters; the array may be NULL), all on the device with no host read; a
 * call without a later backward still updates them.  bn_training = 0 is eval(): the running statistics are read, not
 * written, d_num_batches_tracked and momentum are unused, and d_out is bit-identical to ssb_resnet18_batch's for B
 * <= 1024 (the same conv, finish and head kernels with the same K splits).  The maxpool keeps the index of the element
 * torch's max_pool2d routes the gradient to: the first maximum in row-major window order, a NaN taking the window.
 * 79 launches in training mode, 59 in eval mode, whatever B.
 *
 * ssb_resnet18_train_backward_batch: from d_dpred [B][n_out], the gradient of d_out, and the workspace of the forward
 * with the same arguments and bn_training, writes the gradients of the 20 conv weights, the 20 BatchNorm gamma and
 * beta, and fc's weight and bias; any of them may be NULL (not computed).  The spectrogram gets no gradient.  In
 * training mode the BatchNorm backward has the batch-statistics terms, dx = gamma rstd / N (N dy - sum dy - x^ sum dy
 * x^) per channel, so every row takes part, a row with d_dpred = 0 included; in eval mode it reads the running
 * statistics.  Every sum over rows has a fixed order (channel sums in FP64) and there are no float atomics: two runs
 * give the same bits.  FP32 FMA for the convolutions, no TF32.  With every gradient requested: 115 launches, whatever
 * B and mode.
 *
 * Both: SSB_E_INVALID_ARG for what ssb_resnet18_batch refuses, bn_training not 0 or 1, momentum outside [0, 1], a NULL
 * or misaligned workspace, a misaligned num_batches_tracked counter, and output buffers (d_out, the workspace, the
 * gradients, and in training mode the running statistics and counters) that overlap each other or an input;
 * SSB_E_SHAPE for B > 65535, H or W > 256, fc_in != 512, and in training mode a norm with one value per channel
 * (B H_l W_l == 1, which torch refuses too).  Decided on the host before any launch; B = 0 launches nothing. */
int64_t ssb_resnet18_train_workspace_bytes(int B, int H, int W, int n_out);
int ssb_resnet18_train_forward_batch(ssb_ctx* ctx, int B, const float* d_spec, int H, int W,
                                     const ssb_resnet_conv convs[20], const float* d_fc_weight, const float* d_fc_bias,
                                     int fc_in, int n_out, int bn_training, float momentum,
                                     int64_t* const d_num_batches_tracked[20], float* d_out, void* d_workspace,
                                     void* stream);
int ssb_resnet18_train_backward_batch(ssb_ctx* ctx, int B, const float* d_spec, int H, int W,
                                      const ssb_resnet_conv convs[20], const float* d_fc_weight, int fc_in, int n_out,
                                      int bn_training, const float* d_dpred, void* d_workspace,
                                      float* const d_dweight[20], float* const d_dgamma[20], float* const d_dbeta[20],
                                      float* d_dfc_weight, float* d_dfc_bias, void* stream);

/* One modality of SAVi's visual encoder SMTCNN (ss_baselines/savi/models/smt_cnn.py:17-113) for
 * ssb_smt_cnn_batch.  d_obs: the observation [B][H][W][C] as batch_obs delivers it (observations["rgb"] or
 * ["depth"]); scale 1 multiplies every value by the float32 1 / 255 on load (torch's CUDA x / 255.0, RGB), 0 reads it
 * as is (depth).  resized_h / resized_w and crop_y / crop_x: ResizeCenterCropper(size=(64, 64))'s shortest-edge resize
 * and crop origin (ss_baselines/common/utils.py:341-466), computed by the caller with the reference's own expressions
 * (scale = 64 / min(H, W) in double, resized = int(H scale), int(W scale); crop = resized // 2 - 32); an observation
 * that is already 64 x 64 without a transform is resized 64 x 64, crop (0, 0).  convs: the custom_resnet18's 20 convs
 * as for ssb_smt_resnet18_batch (stem Conv2d(C, 16, 7, 1, 3)); fc = Linear(fc_in = 128 8 8, n_out), d_fc_bias or
 * NULL. */
typedef struct {
    const float* d_obs;
    int32_t C, H, W;
    int32_t scale;
    int32_t resized_h, resized_w, crop_y, crop_x;
    ssb_resnet_conv convs[20];
    const float* d_fc_weight;
    const float* d_fc_bias;
    int32_t fc_in, n_out;
} ssb_smt_cnn_input;

/* SMTCNN.forward under no_grad (rollout time, AudioNavSMTNet.get_features, ss_baselines/savi/ppo/policy.py:439-441)
 * for n_inputs = 1 or 2 modalities in one call: writes d_out[b][...] with input k's n_out features after those of
 * inputs 0 .. k - 1 (torch.cat(cnn_features, dim=1)), row stride the sum of the n_out.
 *
 * One preprocessing launch for all inputs writes a channels-first 64 x 64 image per (input, env): crop pixel (y, x)
 * of channel c is resized pixel (Y, X) = (y + crop_y, x + crop_x), the mean over input rows
 * [floor(Y H / resized_h), ceil((Y + 1) H / resized_h)) and columns [floor(X W / resized_w),
 * ceil((X + 1) W / resized_w)) (adaptive_avg_pool2d, which F.interpolate(mode="area") calls): each scaled value
 * rounded to float32 (x / 255 is materialised before the resize), the values summed in float32 row by row, each row
 * left to right, then divided by the bin's height and then by its width.  The
 * custom_resnet18s then run as in ssb_smt_resnet18_batch, both inputs in the same launches (grid z over inputs), so a
 * call is 39 launches whatever B and n_inputs.  FP32 throughout, no tensor cores, every sum in an order fixed by the
 * layer's shape: an env's features are bit-identical whatever B, its position and whether its modality runs alone or
 * with the other.
 *
 * SSB_E_INVALID_ARG: B < 0, n_inputs outside 1..2, a NULL inputs, a NULL or misaligned d_obs, d_out, fc or conv
 * parameter pointer (d_mean / d_var unused), C < 1, scale not 0 / 1, n_out < 1, eps <= 0.  SSB_E_SHAPE: B > 1024, H or
 * W outside 1..1024, a resize side outside 64..65536, a 64 x 64 crop that does not lie inside the resized image,
 * fc_in != 8192.  All decided on the host before any launch; B = 0 launches nothing.  Scratch, kept by the context
 * for later calls: per input and env 4096 C + 376832 floats (the image, three activation buffers and the K-range
 * partial sums), 1.5 MB; 3.0 GB at B = 1024 for RGB-D. */
int ssb_smt_cnn_batch(ssb_ctx* ctx, int B, int n_inputs, const ssb_smt_cnn_input* inputs, float* d_out, void* stream);

/* SMTCNN trained in the PPO update (AudioNavSMTNet.get_features under grad mode, ss_baselines/savi/ppo/policy.py:439-441,
 * evaluate_actions; the network of ss_baselines/savi/models/smt_cnn.py:17-113): a forward that keeps what the
 * backward needs, and the backward of every parameter.  The inputs table is ssb_smt_cnn_batch's.
 *
 * ssb_smt_cnn_train_workspace_bytes: bytes of the one workspace both entries use (16-byte aligned), or -1 when the
 * arguments or shape are refused.  It holds each input's 64 x 64 image, then per input the layout of
 * ssb_smt_resnet18_train_workspace_bytes (saved pre-norm sums, GroupNorm statistics, stem, conv1 and block outputs,
 * then the backward's scratch), without labels: about 6.06 MB per RGB row and 6.03 MB per depth row, 7.26 GB at B =
 * 600 for RGB-D.  The
 * forward writes it, the backward reads it and overwrites the scratch parts, so a backward needs the workspace of its
 * own forward, untouched in between.
 *
 * ssb_smt_cnn_train_forward_batch: d_out as ssb_smt_cnn_batch's ([B][sum n_out], inputs side by side), with B <= 65535
 * instead of 1024.  One cnn_prep_kernel launch writes every input's image into the workspace, then each network runs
 * ssb_smt_resnet18_train_forward_batch's launches (the rollout's conv, finish and head kernels with the same K
 * splits, the finish also saving its sums and statistics), one network after the other.  So d_out is bit-identical to
 * ssb_smt_cnn_batch's for every row at any B and row order.  1 + 38 n_inputs launches, whatever B.
 *
 * ssb_smt_cnn_train_backward_batch: from d_dout [B][sum n_out], the gradient of d_out (each network reads its own
 * columns, row stride sum n_out), and the workspace of the forward with the same arguments, writes per input k the
 * 62 gradients d_grads[62 k ..]: the 20 conv weights, the 20 GroupNorm gammas, the 20 betas, fc's weight and bias, in
 * the order of the parameters' conv table; any may be NULL (not computed).  The observations get no gradient.  Per
 * network ssb_smt_resnet18_train_backward_batch's kernels: rows with an all-zero d_dout slice of that network are
 * dropped on the device, every sum over rows runs in list order, and the stem's dW is a GEMM over all C channels of
 * the saved image.  FP32 FMA, no TF32 and no float atomics: two runs give the same bits, and a batch's gradients equal
 * those of the same batch without its silent rows.  With every gradient requested: 80 launches per input, whatever B
 * and the number of live rows.
 *
 * Both: SSB_E_INVALID_ARG for what ssb_smt_cnn_batch refuses, a NULL or misaligned workspace, a NULL d_grads table,
 * and output buffers (d_out, the workspace, the gradients) that overlap each other or an input; SSB_E_SHAPE for B >
 * 65535 and the shapes ssb_smt_cnn_batch refuses.  Decided on the host before any launch; B = 0 launches nothing. */
int64_t ssb_smt_cnn_train_workspace_bytes(int B, int n_inputs, const ssb_smt_cnn_input* inputs);
int ssb_smt_cnn_train_forward_batch(ssb_ctx* ctx, int B, int n_inputs, const ssb_smt_cnn_input* inputs, float* d_out,
                                    void* d_workspace, void* stream);
int ssb_smt_cnn_train_backward_batch(ssb_ctx* ctx, int B, int n_inputs, const ssb_smt_cnn_input* inputs,
                                     const float* d_dout, void* d_workspace, float* const* d_grads, void* stream);

/* A Linear's parameters, torch's layout: d_weight [out][in], d_bias [out]. */
typedef struct {
    const float* d_weight;
    const float* d_bias;
} ssb_linear;

/* An affine LayerNorm over the last dim: d_gamma / d_beta [d_model], eps > 0. */
typedef struct {
    const float* d_gamma;
    const float* d_beta;
    float eps;
    int32_t reserved;
} ssb_layer_norm;

/* SMTStateEncoder (ss_baselines/savi/models/smt_state_encoder.py) with one encoder and one decoder layer of its
 * nn.Transformer (post-norm, ReLU, dim_feedforward = d_model, final encoder.norm and decoder.norm).  d_in: the token
 * width D; pose_index: _pose_indices[0], or -1 without pose encoding; pretraining: _pretraining (0 or 1).  pose =
 * pose_encoder Linear(5, 16) (unused when pose_index < 0); fuse1 / fuse2: fusion_encoder[0] / [2], with fuse1 taking
 * pose_index + 16 features (d_in without pose encoding).  enc_qkv / dec_sa_qkv / dec_ca_qkv: a MultiheadAttention's
 * in_proj ([3 d_model][d_model] weight, [3 d_model] bias; only the V rows of dec_sa_qkv are read); enc_out / dec_sa_out /
 * dec_ca_out: its out_proj; *_ff1 / *_ff2: linear1 / linear2; enc_norm1/2, dec_norm1/2/3: the layers' norms; enc_norm /
 * dec_norm: transformer.encoder.norm / decoder.norm. */
typedef struct {
    int32_t d_in, pose_index, d_model, n_heads, pretraining;
    ssb_linear pose, fuse1, fuse2;
    ssb_linear enc_qkv, enc_out, enc_ff1, enc_ff2;
    ssb_layer_norm enc_norm1, enc_norm2, enc_norm;
    ssb_linear dec_sa_qkv, dec_sa_out, dec_ca_qkv, dec_ca_out, dec_ff1, dec_ff2;
    ssb_layer_norm dec_norm1, dec_norm2, dec_norm3, dec_norm;
} ssb_smt_params;

/* Bytes of device scratch ssb_smt_state_encoder_batch needs for B envs and M memory slots: 5 B (M + 1) d_model floats
 * of per-token activations after B per-env counts (4 B bytes, rounded up to a multiple of 256).  -1 for a NULL p, B < 0, M < 0 or d_model < 1. */
int64_t ssb_smt_scratch_bytes(int B, int M, const ssb_smt_params* p);

/* SMTStateEncoder.single_forward(x, memory, memory_masks, goal) at rollout time (under no_grad),
 * ss_baselines/savi/models/smt_state_encoder.py:92-157 with _encode_pose :179-245, as called by
 * AudioNavSMTNet.forward, ss_baselines/savi/ppo/policy.py:380-403.  d_x [B][d_in], d_memory [M][B][d_in], d_masks
 * [B][M] float (slot j of env b is valid iff !((1 - mask) > 0); none under pretraining; the current token always),
 * d_goal [B][d_model] or NULL (the decoder's target is then the fused current token), d_out [B][d_model].  Only valid
 * tokens are read and computed: a masked slot's memory row is never read, so NaN or Inf there has no effect (the
 * reference multiplies its zero attention weight by it).  FP32 FMA throughout, no tensor cores; every sum has an order
 * fixed by the layer's shape, so an env's output is bit-identical whatever B, its position and its masked slots.
 * Parameters are read through the pointers on every call.  6 launches per call, whatever B, M and the masks; the host
 * never reads the masks.  d_scratch: ssb_smt_scratch_bytes(B, M, p) bytes, 16-byte aligned.  SSB_E_INVALID_ARG: a
 * NULL or misaligned pointer (d_memory and d_masks may be NULL when M = 0), B < 0, M < 0, d_in < 1, pose_index < -1,
 * n_heads < 1, d_model % n_heads != 0, pretraining not 0 / 1, eps <= 0.  SSB_E_SHAPE: B > 1024, M + 1 > 1024,
 * d_model > 512, d_model / n_heads > 128, d_in > 1024, pose_index >= 0 and pose_index + 4 > d_in.  Both decided on the host before any
 * launch; B = 0 launches nothing. */
int ssb_smt_state_encoder_batch(ssb_ctx* ctx, int B, int M, const float* d_x, const float* d_memory,
                                const float* d_masks, const float* d_goal, const ssb_smt_params* p, void* d_scratch,
                                float* d_out, void* stream);

/* SMTStateEncoder.single_forward for training (PPO's evaluate_actions, grad enabled),
 * ss_baselines/savi/models/smt_state_encoder.py:92-157 with _encode_pose :179-245: a forward that keeps what its
 * backward reads in a workspace, and that backward.  Both take the inputs and the ssb_smt_params of
 * ssb_smt_state_encoder_batch, with the same meaning.
 *
 * ssb_smt_train_workspace_bytes: bytes of the workspace for B rows and M memory slots, or -1 for a NULL p, B < 0, B >
 * 65535, M < 0, M + 1 > 1024, d_model < 1, n_heads < 1, d_in < 1 or > 1024, pose_index < -1.  Per-token activations,
 * gradients and partial sums, about 33 B (M + 1) d_model floats (6.14 GB at B 600, M 300, d_model 256).
 *
 * ssb_smt_state_encoder_train_forward_batch: the six launches of ssb_smt_state_encoder_batch through the same host
 * code, on workspace buffers that nothing overwrites, plus the values those kernels otherwise keep only in shared
 * memory (compacted slots, fusion input and hidden ReLU, the tail's LayerNorm inputs and statistics, its FF hidden
 * ReLU).  d_out [B][d_model] is bit-identical to ssb_smt_state_encoder_batch for B <= 1024, and above that to it run
 * in chunks of 1024 rows (rows are independent).  Limits and error codes as ssb_smt_state_encoder_batch, with the
 * workspace (16-byte aligned) as d_scratch and 1 <= B <= 65535.
 *
 * ssb_smt_state_encoder_train_backward_batch: from the workspace of a forward with the same arguments and parameter
 * values, and d_dout [B][ld_dout] (ld_dout >= d_model), the gradient of sum(out * dout):
 *   d_grads: every parameter's gradient in ssb_smt_params order (pose.weight, pose.bias first with pose encoding,
 *            then fuse1 .. enc_ff2, enc_norm1 .. enc_norm gamma / beta, dec_sa_qkv .. dec_ff2, dec_norm1 .. dec_norm):
 *            40 pointers with pose encoding, 38 without, each in its parameter's shape; a NULL entry is not computed.
 *            dec_sa_qkv's Q and K rows get exactly 0 (self-attention over one key).
 *   d_dx [B][d_in] (NULL: not computed): feature columns from the current token; with pose encoding, the agent's
 *            x, y and heading through every valid token's relative pose and its time through its own token (0 through
 *            the distance and the bearing at distance 0, as torch's autograd gives), 0 past pose_index + 4.
 *   d_dgoal [B][d_model] (NULL: not computed; needs d_goal).
 * Memory and masks get no gradient.  FP32 FMA, no atomics: every weight gradient is a sum over rows and valid tokens
 * in a fixed order (32 row splits by env, then the splits in order), so two calls give the same bits.  Masked slots
 * are never read.  10 launches whatever B, M and the masks; no host synchronisation.  SSB_E_INVALID_ARG also for a
 * NULL d_grads, ld_dout < d_model, misaligned gradients, d_dgoal without d_goal.  Decided on the host before any
 * launch; B = 0 launches nothing. */
int64_t ssb_smt_train_workspace_bytes(int B, int M, const ssb_smt_params* p);
int ssb_smt_state_encoder_train_forward_batch(ssb_ctx* ctx, int B, int M, const float* d_x, const float* d_memory,
                                              const float* d_masks, const float* d_goal, const ssb_smt_params* p,
                                              void* d_workspace, float* d_out, void* stream);
int ssb_smt_state_encoder_train_backward_batch(ssb_ctx* ctx, int B, int M, const float* d_x, const float* d_memory,
                                               const float* d_masks, const float* d_goal, const ssb_smt_params* p,
                                               const float* d_dout, int ld_dout, void* d_workspace,
                                               float* const* d_grads, float* d_dx, float* d_dgoal, void* stream);

/* AV-WaN's geometric, acoustic and action maps kept on the device (ss_baselines/av_wan/models/mapper.py, Planner
 * .add_maps_to_observation at planner.py:76-83).  Env workers keep running the reference Mapper for the planner's
 * graph and send map-update records instead of maps; ssb_map_update_batch replays a step's records into per-slot
 * device maps and ssb_map_observe_batch crops the three egocentric observations from them.
 *
 * Geometry (one per call, shared by every slot of the state buffers):
 *   N = internal_size (GEOMETRIC_MAP.INTERNAL_MAP_SIZE), s = stride (int(ACTION_MAP.MAP_RESOLUTION /
 *   GEOMETRIC_MAP.MAP_RESOLUTION)), S = map_size (GEOMETRIC_MAP.MAP_SIZE, even), a = action_size (ACTION_MAP.MAP_SIZE,
 *   odd), E = ego_size (the E x E x 2 ego map), M = N / s (integer division: the acoustic map's side),
 *   encoding SSB_MAP_INTENSITY or SSB_MAP_AVERAGE_INTENSITY (ACOUSTIC_MAP.ENCODING), acoustic 0 / 1
 *   (use_acoustic_map: with 0 no acoustic map is kept and d_amap may be NULL), n_slots = slots in the state buffers.
 *   Limits: 1 <= N <= SSB_MAP_MAX_INTERNAL, 1 <= s <= N, 2 <= S <= SSB_MAP_MAX_INTERNAL, 1 <= a <= SSB_MAP_MAX_EGO,
 *   1 <= E <= min(N, SSB_MAP_MAX_EGO), 1 <= n_slots <= SSB_MAP_MAX_SLOTS.
 * State (caller-owned, zeroed or reset before first use):
 *   d_gmap: uint8 [n_slots][SSB_MAP_PITCH(N)], 16-byte aligned; cell (row y, col x) of slot k is byte
 *           k * SSB_MAP_PITCH(N) + y N + x, bit 0 = channel 0 (obstacle), bit 1 = channel 1 (explored);
 *   d_amap: float64 [n_slots][M][M], 8-byte aligned, the reference's acoustic map (channel 0).
 * Orientation is in degrees, one of 0, 90, 180, 270; the map is viewed rotated by k = ((orientation - 270) mod 360)
 * / 90 quarter turns, np.rot90(map, k), as the reference's rotate_map(map, -self._rotation) does. */
#define SSB_MAP_INTENSITY 0
#define SSB_MAP_AVERAGE_INTENSITY 1
#define SSB_MAP_RESET 0
#define SSB_MAP_UPDATE 1
#define SSB_MAP_MAX_SLOTS 65535
#define SSB_MAP_MAX_INTERNAL 4096
#define SSB_MAP_MAX_EGO 255
#define SSB_MAP_AM_CROP 20      /* get_egocentric_acoustic_map()'s default crop_map_size, whatever ACOUSTIC_MAP.MAP_SIZE */
#define SSB_MAP_PITCH(n) ((((int64_t)(n) * (n)) + 15) & ~(int64_t)15)

typedef struct {
    int32_t internal_size, stride, map_size, action_size, ego_size, encoding, acoustic, n_slots;
} ssb_map_geometry;

/* One Mapper.reset (kind SSB_MAP_RESET: only slot is read) or one completed Mapper.update (SSB_MAP_UPDATE). */
typedef struct {
    int32_t slot, kind;
    int32_t x, y, orientation;  /* the mapper's pose after the update */
    int32_t reserved;           /* ssb_map_update_device_intensity_batch: index into d_intensity; otherwise unused */
    double intensity;         /* float64(intensity) as the reference stores it */
    double half;                /* 0.5 * intensity as the reference evaluates it, widened to float64 */
    int64_t ego_offset;         /* first byte of np.packbits(ego_map > 0.5) ([E][E][2], MSB first) in h_ego */
} ssb_map_record;

/* Applies n_records records in ONE launch (nothing for n_records = 0).  Records of one slot apply in array order,
 * different slots in parallel (one CTA per slot touched).  Reset: the slot's geometric and acoustic maps become 0.
 * Update, with (rx, ry) the pose in the rotated view: ORs the ego bits into rows [ry - E, ry) and columns
 * [rx - E/2, rx - E/2 + E) of the rotated view (Mapper.update's window; nothing at E = 1 and ry = 0, where the
 * reference's slice is empty), then clears channel 0 of the agent's cell when rx and ry are at most N + 1 - s (the
 * reference's "marked current position as obstacle" branch: its loop visits that cell, which the window never covers,
 * unless it stands within s - 1 cells of the rotated view's far edges); with an acoustic map, cell (y / s, x / s)
 * becomes intensity (SSB_MAP_INTENSITY) or, for SSB_MAP_AVERAGE_INTENSITY, intensity if it is 0 (or -0) and
 * half + 0.5 * cell in float64 without contraction otherwise.
 * h_records and h_ego are host memory; they are staged through a context-owned pinned buffer and may be reused when
 * the call returns.  SSB_E_INVALID_ARG: a NULL or misaligned state pointer, n_records < 0, NULL h_records, bad
 * geometry (limits above, odd S, even a, unknown encoding), a slot outside [0, n_slots), an unknown kind, an
 * orientation not a multiple of 90 in [0, 360), ego bits outside [0, ego_bytes).  SSB_E_SHAPE: an update whose window
 * leaves the internal map (E = 1 at ry = 0 excepted) or whose pose lies outside it (the reference raises there), at
 * s = 1 an update with ry = N - 1 or rx - E/2 + E >= N - 1 (the reference's loop then reads row or column N and raises
 * IndexError), or an acoustic cell outside the M x M map.  All decided on the host before any launch. */
int ssb_map_update_batch(ssb_ctx* ctx, const ssb_map_geometry* g, uint8_t* d_gmap, double* d_amap, int n_records,
                         const ssb_map_record* h_records, const uint8_t* h_ego, int64_t ego_bytes, void* stream);

/* ssb_map_update_batch with the acoustic values already on the device (env workers that defer the Intensity sensor to
 * the trainer): with an acoustic map, every update record takes v = d_intensity[reserved] (float32, e.g. the output of
 * ssb_intensity_batch) instead of its intensity and half fields and applies intensity = (double)v and half = 0.5 *
 * (double)v in float64 -- what a worker computes from the Python float the sensor returns in process.  (The
 * reference's np.float32 intensity gives a float32 product instead; the two differ only where 0.5 v is subnormal in
 * float32.)  Resets, and every record without an acoustic map, read no intensity.  SSB_E_INVALID_ARG: everything
 * ssb_map_update_batch refuses, n_intensity < 0, and, for a record that indexes it, a NULL or misaligned d_intensity
 * or an index outside [0, n_intensity).  All decided on the host before any launch. */
int ssb_map_update_device_intensity_batch(ssb_ctx* ctx, const ssb_map_geometry* g, uint8_t* d_gmap, double* d_amap,
                                          int n_records, const ssb_map_record* h_records, const uint8_t* h_ego,
                                          int64_t ego_bytes, const float* d_intensity, int64_t n_intensity,
                                          void* stream);

/* Writes the egocentric maps of B envs in ONE launch (nothing for B = 0).  h_poses: host int32 [B][4] = (slot, x, y,
 * orientation); h_tables: host int32 [4][2][L] = for each k the sorted rotated navigable xs, then ys (Mapper.
 * compute_navigable_xys, computed once by the caller; any values in [0, N)).  Any output may be NULL:
 *   d_gm [B][gm_stride] floats, row b = (S, S, 2): get_egocentric_geometric_map, 0 outside the internal map;
 *   d_am [B][am_stride] floats, row b = (20, 20, 1): get_egocentric_acoustic_map(), 0 outside the acoustic map;
 *   d_action [B][action_stride] floats, row b = (a, a, 1): 1 - grid_map[gy - a/2 : gy + a/2 + 1, gx - a/2 : ..., 0] of
 *   get_egocentric_occupancy_map, grid_map = view[ys_k][:, xs_k], gx = rx / s, gy = ry / s.
 * Each value is the reference's float64 value rounded to float32.  Strides are in floats, at least the row size.
 * SSB_E_INVALID_ARG: bad geometry, B < 0 or > SSB_MAP_MAX_SLOTS, NULL h_poses, a NULL or misaligned state pointer a
 * requested output needs, a misaligned output, a short stride, L < 1 or a table entry outside [0, N) when the action
 * map is requested, a slot outside [0, n_slots), a bad orientation.  SSB_E_SHAPE: a pose outside the internal map, an
 * acoustic cell outside the M x M map (d_am requested), an occupancy window that leaves the L x L grid (the reference
 * returns a wrongly shaped array there).  All decided on the host before any launch. */
int ssb_map_observe_batch(ssb_ctx* ctx, const ssb_map_geometry* g, const uint8_t* d_gmap, const double* d_amap, int B,
                          const int32_t* h_poses, const int32_t* h_tables, int L, float* d_gm, int64_t gm_stride,
                          float* d_am, int64_t am_stride, float* d_action, int64_t action_stride, void* stream);

/* Remote env workers' RGB and depth frames (soundspaces_b200.frames): a step's visual observations gathered from
 * device frame banks into float32 rows, for up to SSB_FRAME_MAX_SENSORS sensors in ONE launch.  Per sensor, d_bank
 * holds bank_rows rows of row_elems elements of dtype (uint8 RGB or float32 depth, as the sensor produced them) and
 * d_stage the n_fill rows uploaded for this call.  Destination row i (i < N) of d_dst, dst_stride floats after row
 * i - 1, receives the row h_index[i] names: bank row h_index[i] when >= 0, staged row -1 - h_index[i] otherwise;
 * uint8 becomes float32 exactly (as torch's .float()), float32 is copied bit for bit.  Staged row j is also written
 * to bank row h_fill[j].  h_index and h_fill are host int32 arrays packed into the launch's parameters.  16-byte
 * loads and stores where every pointer, the row and the stride allow.  N = 0 launches nothing.
 * SSB_E_INVALID_ARG: n_sensors outside [1, SSB_FRAME_MAX_SENSORS], N < 0, an unknown dtype, row_elems < 1,
 * bank_rows < 1, dst_stride < row_elems, n_fill outside [0, N], a NULL pointer the call needs, a float32 pointer not
 * aligned to 4 bytes, an index outside [-n_fill, bank_rows), a fill row outside [0, bank_rows) or filled twice, an
 * index naming a bank row the call fills, a destination or a filled bank sharing bytes with any other buffer of the
 * call.  SSB_E_SHAPE: N > SSB_FRAME_MAX_N, a bank or destination of 2^46 bytes or more.  All decided on the host
 * before any launch. */
#define SSB_FRAME_MAX_SENSORS 4
#define SSB_FRAME_MAX_N 256
#define SSB_FRAME_U8 0
#define SSB_FRAME_F32 1
typedef struct {
    void* d_bank;
    const void* d_stage;
    float* d_dst;
    const int32_t* h_index;     /* [N] */
    const int32_t* h_fill;      /* [n_fill] */
    int64_t row_elems;
    int64_t bank_rows;
    int64_t dst_stride;         /* floats */
    int32_t n_fill;
    int32_t dtype;              /* SSB_FRAME_U8 or SSB_FRAME_F32 */
} ssb_frame_sensor;
int ssb_frame_gather_batch(ssb_ctx* ctx, int n_sensors, const ssb_frame_sensor* sensors, int N, void* stream);

/* PCM helpers.  decode: float32(x) / 32768 (exact).  encode mode 0: round(x*32768) saturated;
 * mode 1: trunc(x*32767) saturated (interactive_demo.py:110). */
int ssb_pcm16_decode(ssb_ctx* ctx, const int16_t* d_in, int64_t n, float* d_out, void* stream);
int ssb_pcm16_encode(ssb_ctx* ctx, const float* d_in, int64_t n, int mode, int16_t* d_out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SSB200_H */
