"""-m gpu: the reference's session state behind the operator hook.  falcon_main's --prompt-cache saves and loads the context through
llama_save_session_file / llama_load_session_file; their KV section is copied by ggml_cpy graphs over views of the host cache
(falcon_copy_state_data / falcon_set_state_data, libfalcon.cpp:4226-4470).  Under the whole-graph takeover the cache lives in HBM, so the
hook serves those copies from the device: a save is the device cache, a load goes into it, and a first eval after a load (at n_past > 0)
is taken over like one at 0.  Each test pairs the reference behind the hook with a standalone b200_falcon loaded from the same file
(tests/test_surface_nodes_gpu.py holds takeover to that engine bit for bit)."""
import ctypes as C
import os
import struct
import numpy as np
import pytest
import pyoracle as po
from helpers import TINY_40B, TINY_7B, synth_model, ggcc

pytestmark = pytest.mark.gpu
HOOK = os.path.join(po.HERE, "_ref", "libfalcon_hook.so")
CPU_REF = os.path.join(po.HERE, "_ref", "libfalcon_ref.so")
need_hook = pytest.mark.skipif(not os.path.exists(HOOK), reason="oracle/_ref/libfalcon_hook.so not present (built by make -C oracle ref from the reference sources)")

# Falcon-40B / 180B's KV row: n_head_kv 8, 512 floats per position and layer
TINY_40B_KV8 = dict(n_vocab=512, n_embd=1024, n_head=16, n_head_kv=8, n_layer=2, falcon_type=40)
MODELS = [(TINY_40B, po.Q4_K, 15), (TINY_7B, po.Q4_0, 2), (TINY_40B_KV8, po.Q4_K, 15)]
IDS = ["40b-q4_K", "7b-q4_0", "40b-kv8-q4_K"]
N_CTX = 64
PROMPT = np.array([11] + list(range(100, 111)), np.int32)
# falcon_main's order: BOS warm-up at 0, the prompt at 0 (the GEMM), decode steps -> a 15-position session
SAVE_SEQ = [(np.array([11], np.int32), 0), (PROMPT, 0)] + [(np.array([300 + i], np.int32), 12 + i) for i in range(3)]
N_SAVED = 15
# what a --prompt-cache run continues with: one token at 15 (the first eval of the new context), a 10-token batch, decode steps
RESUME_SEQ = [(np.array([400], np.int32), 15), (np.arange(120, 130, dtype=np.int32), 16)] + \
             [(np.array([500 + i], np.int32), 26 + i) for i in range(3)]


class SessionRef(po.RefFalcon):
    """RefFalcon plus the reference's own session calls (libfalcon.h:194, 213-214), called straight through ctypes"""

    def __init__(self, path, hook=True):
        super().__init__(path, n_ctx=N_CTX, n_batch=64, logits_all=True, hook=hook, n_gpu_layers=99 if hook else 0)
        self.L.llama_save_session_file.restype = C.c_bool
        self.L.llama_save_session_file.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p, C.c_size_t]
        self.L.llama_load_session_file.restype = C.c_bool
        self.L.llama_load_session_file.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
        self.L.llama_get_kv_cache_token_count.restype = C.c_int
        self.L.llama_get_kv_cache_token_count.argtypes = [C.c_void_p]

    def save_session(self, path, tokens):
        t = np.ascontiguousarray(tokens, np.int32)
        assert self.L.llama_save_session_file(self.h, str(path).encode(), t.ctypes.data, t.size)

    def load_session(self, path):
        """-> the session's tokens"""
        t, n = np.zeros(N_CTX, np.int32), C.c_size_t(0)
        assert self.L.llama_load_session_file(self.h, str(path).encode(), t.ctypes.data, t.size, C.byref(n))
        return t[:n.value]

    def kv_ntok(self):
        return self.L.llama_get_kv_cache_token_count(self.h)


def kv_section(path, hp):
    """-> (kv_ntok, K [n_layer][n][E], V [n_layer][n][E]) of a session file (llama_save_session_file, falcon_copy_state_data; V is
    stored transposed, [n_layer][E][n])"""
    b = open(path, "rb").read()
    assert struct.unpack_from("<II", b, 0) == (0x6767736E, 1)
    o = 8 + 9 * 4                                             # falcon_hparams: eight int32 and the ftype enum
    o += 4 + 4 * struct.unpack_from("<I", b, o)[0]            # the tokens
    o += 8 + 64 * 1024                                        # rng: size and LLAMA_MAX_RNG_STATE bytes
    cap = struct.unpack_from("<Q", b, o)[0]; o += 16 + 4 * cap
    o += 8 + 4 * struct.unpack_from("<Q", b, o)[0]            # embeddings
    kv_size, n = struct.unpack_from("<Qi", b, o); o += 12
    L, E = hp["n_layer"], hp["n_head_kv"] * 64
    assert kv_size > 0 and len(b) == o + 2 * L * n * E * 4
    K = np.frombuffer(b, np.float32, L * n * E, o).reshape(L, n, E)
    V = np.frombuffer(b, np.float32, L * n * E, o + L * n * E * 4).reshape(L, E, n).transpose(0, 2, 1)
    return n, K, V


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _model(tmp_path, hp, wt, ftype):
    path = str(tmp_path / "m.ggcc")
    ggcc.write_ggcc(path, hp, synth_model(hp, wt, seed=1234), ftype=ftype)
    return path


def _engine(gpu, path):
    eng = gpu.Falcon(gpu.Falcon.read_hparams(path), n_ctx=N_CTX, n_batch=512)
    eng.load_ggcc(path)
    return eng


def _tokens(seq):
    return np.concatenate([t for t, _ in seq])


def _loose(got, want, S):
    """DESIGN §2's bound for the prompt GEMM path: every session here holds rows a 12-token batch wrote through fp16 operands"""
    d = np.abs(got - want)
    assert d.max() <= 3e-2 * S and np.median(d) <= 5e-3 * S, (float(d.max()), float(np.median(d)), S)


def _hook_saves(gpu, path, sess, eng=None):
    """SAVE_SEQ behind the hook (and on `eng`, if given), then a session file; the hook context is closed"""
    ref = SessionRef(path)
    try:
        for toks, n_past in SAVE_SEQ:
            ref.eval(toks, n_past, n_threads=2)
            if eng is not None:
                eng.eval(toks, n_past, n_ctx_rope=N_CTX, all_logits=True)
        assert ref.kv_ntok() == N_SAVED
        ref.save_session(sess, _tokens(SAVE_SEQ))
    finally:
        ref.close()


@need_hook
@pytest.mark.parametrize("hp,wt,ftype", MODELS, ids=IDS)
def test_save_is_the_device_cache(gpu, tmp_path, monkeypatch, hp, wt, ftype):
    monkeypatch.delenv("B200_NO_TAKEOVER", raising=False)
    path, sess = _model(tmp_path, hp, wt, ftype), str(tmp_path / "s.bin")
    eng = _engine(gpu, path)
    try:
        t0 = gpu.lib().b200_surface_takeover_evals()
        _hook_saves(gpu, path, sess, eng)
        assert gpu.lib().b200_surface_takeover_evals() - t0 == len(SAVE_SEQ) - 1
        n, K, V = kv_section(sess, hp)
        assert n == N_SAVED
        for layer in range(hp["n_layer"]):
            k, v = eng.kv_read(layer, 0, n)
            assert np.array_equal(bits(K[layer]), bits(k)), layer
            assert np.array_equal(bits(V[layer]), bits(v)), layer
    finally:
        eng.free()


@need_hook
@pytest.mark.parametrize("hp,wt,ftype", MODELS, ids=IDS)
def test_load_resumes_on_the_device(gpu, tmp_path, monkeypatch, hp, wt, ftype):
    """a fresh context loads the session and evaluates at 15 without a warm-up (falcon_main.cpp:662-673): that first eval runs through
    the per-node path, the engine then imports the 15 restored positions, and every later eval is the standalone engine's, bit for bit"""
    monkeypatch.delenv("B200_NO_TAKEOVER", raising=False)
    path, sess = _model(tmp_path, hp, wt, ftype), str(tmp_path / "s.bin")
    eng = _engine(gpu, path)
    lib = gpu.lib()
    try:
        _hook_saves(gpu, path, sess, eng)
        ref = SessionRef(path)
        try:
            assert np.array_equal(ref.load_session(sess), _tokens(SAVE_SEQ)) and ref.kv_ntok() == N_SAVED
            for i, (toks, n_past) in enumerate(RESUME_SEQ):
                taken = lib.b200_surface_takeover_evals()
                got = ref.eval(toks, n_past, n_threads=2)
                want = eng.eval(toks, n_past, n_ctx_rope=N_CTX, all_logits=True)
                if i == 0:
                    assert lib.b200_surface_takeover_evals() == taken
                    _loose(got, want, float(np.abs(want).max()))
                    continue
                assert lib.b200_surface_takeover_evals() == taken + 1, (i, n_past)
                d = np.flatnonzero(bits(got) != bits(want))
                assert d.size == 0, "eval %d (N %d at n_past %d): %d logits differ" % (i, toks.size, n_past, d.size)
        finally:
            ref.close()
    finally:
        eng.free()


@need_hook
@pytest.mark.parametrize("hp,wt,ftype", MODELS, ids=IDS)
def test_restore_into_a_running_takeover(gpu, tmp_path, monkeypatch, hp, wt, ftype):
    """prompt A, save, prompt B over it, load A's session: the decode steps that follow are A's own continuation, bit for bit.
    37 positions: the transposes run over a partial second tile"""
    monkeypatch.delenv("B200_NO_TAKEOVER", raising=False)
    path, sess = _model(tmp_path, hp, wt, ftype), str(tmp_path / "a.bin")
    A = np.array([11] + list(range(100, 136)), np.int32)
    B = np.array([11] + list(range(200, 236)), np.int32)
    steps = [(np.array([300 + i], np.int32), A.size + i) for i in range(4)]
    eng = _engine(gpu, path)
    lib = gpu.lib()
    ref = SessionRef(path)
    try:
        t0 = lib.b200_surface_takeover_evals()
        for toks, n_past in [(np.array([11], np.int32), 0), (A, 0)]:
            ref.eval(toks, n_past, n_threads=2)
            eng.eval(toks, n_past, n_ctx_rope=N_CTX, all_logits=True)
        ref.save_session(sess, A)
        ref.eval(B, 0, n_threads=2)
        assert np.array_equal(ref.load_session(sess), A) and ref.kv_ntok() == A.size
        for toks, n_past in steps:
            got = ref.eval(toks, n_past, n_threads=2)
            want = eng.eval(toks, n_past, n_ctx_rope=N_CTX, all_logits=True)
            d = np.flatnonzero(bits(got) != bits(want))
            assert d.size == 0, "decode at n_past %d: %d logits differ" % (n_past, d.size)
        assert lib.b200_surface_takeover_evals() - t0 == 2 + len(steps)       # A, B and the steps; the warm-up was the learning eval
    finally:
        ref.close()
        eng.free()


def _continue(ref, seq):
    return [ref.eval(toks, n_past, n_threads=2) for toks, n_past in seq]


@need_hook
@pytest.mark.skipif(not os.path.exists(CPU_REF), reason="oracle/_ref/libfalcon_ref.so not present")
@pytest.mark.parametrize("hp,wt,ftype", MODELS[:2], ids=IDS[:2])
def test_sessions_move_between_the_cpu_build_and_the_hook(gpu, tmp_path, monkeypatch, hp, wt, ftype):
    """a session saved by the CPU reference continues behind the hook, and one saved behind the hook continues in the CPU reference,
    both within the loose bound of the CPU reference's own continuation"""
    monkeypatch.delenv("B200_NO_TAKEOVER", raising=False)
    path, sess_cpu, sess_hook = _model(tmp_path, hp, wt, ftype), str(tmp_path / "cpu.bin"), str(tmp_path / "hook.bin")
    lib = gpu.lib()
    cpu = SessionRef(path, hook=False)
    try:
        _continue(cpu, SAVE_SEQ)
        cpu.save_session(sess_cpu, _tokens(SAVE_SEQ))
        truth = _continue(cpu, RESUME_SEQ)
    finally:
        cpu.close()
    S = max(float(np.abs(t).max()) for t in truth)
    # CPU -> hook: the first eval is the learning one, every later one is taken over
    ref = SessionRef(path)
    try:
        ref.load_session(sess_cpu)
        t0 = lib.b200_surface_takeover_evals()
        got = _continue(ref, RESUME_SEQ)
        assert lib.b200_surface_takeover_evals() - t0 == len(RESUME_SEQ) - 1
    finally:
        ref.close()
    for g, w in zip(got, truth):
        _loose(g, w, S)
    # hook -> CPU
    _hook_saves(gpu, path, sess_hook)
    cpu = SessionRef(path, hook=False)
    try:
        cpu.load_session(sess_hook)
        assert cpu.kv_ntok() == N_SAVED
        got = _continue(cpu, RESUME_SEQ)
    finally:
        cpu.close()
    for g, w in zip(got, truth):
        _loose(g, w, S)


@need_hook
@pytest.mark.parametrize("hp,wt,ftype", MODELS[:2], ids=IDS[:2])
def test_per_node_path_keeps_the_host_session(gpu, tmp_path, monkeypatch, hp, wt, ftype):
    """B200_NO_TAKEOVER=1: save and load go through the host buffers, nothing is taken over, and the loaded context continues within
    the loose bound of the saving context's own continuation"""
    monkeypatch.setenv("B200_NO_TAKEOVER", "1")
    path, sess = _model(tmp_path, hp, wt, ftype), str(tmp_path / "s.bin")
    lib = gpu.lib()
    t0 = lib.b200_surface_takeover_evals()
    ref = SessionRef(path)
    try:
        _continue(ref, SAVE_SEQ)
        ref.save_session(sess, _tokens(SAVE_SEQ))
        truth = _continue(ref, RESUME_SEQ)
    finally:
        ref.close()
    ref = SessionRef(path)
    try:
        ref.load_session(sess)
        got = _continue(ref, RESUME_SEQ)
    finally:
        ref.close()
    assert lib.b200_surface_takeover_evals() == t0
    S = max(float(np.abs(t).max()) for t in truth)
    for g, w in zip(got, truth):
        _loose(g, w, S)
