// Package sbvverifier implements SmartBFT's api.Verifier on top of libsbv.so (include/sbv.h).
//
// UNBUILT AND UNTESTED: there is no Go toolchain in the build image. The same logic is built and
// tested in C++ (consensus_b200/host/verifier.hpp, callsites.hpp); this file is the mechanical Go
// rendering a maintainer would start from.
//
// Reference interface: pkg/api/dependencies.go:54-71. Signed-bytes convention: INTEGRATION.md.
package sbvverifier

/*
#cgo CFLAGS: -I${SRCDIR}/../../../include
#cgo LDFLAGS: -L${SRCDIR}/../../../consensus_b200 -lsbv
#include <stdlib.h>
#include "sbv.h"
*/
import "C"

import (
	"bytes"
	"encoding/binary"
	"encoding/hex"
	"errors"
	"fmt"
	"sync"
	"time"
	"unsafe"

	"github.com/hyperledger-labs/SmartBFT/pkg/types"
)

// item is one unit of engine work: verify (r, s) under registry slot `slot` over SHA-256(msg), or, when ed is set,
// the Ed25519 signature edSig under slot `slot` of the Ed25519 registry over msg (crypto/ed25519.Verify). When keyed
// is set the key travels with the item instead of a slot: key = P-256 X || Y, or the Ed25519 key in key[:32].
type item struct {
	r, s  [32]byte
	slot  uint32
	msg   []byte
	ed    bool
	edSig [64]byte
	keyed bool
	key   [64]byte
}

// clientKey is a client key kept on the host (WithClientKeysPerItem): P-256 X || Y, or an Ed25519 key in key[:32].
type clientKey struct {
	ed  bool
	key [64]byte
}

// Option configures a Verifier at New.
type Option func(*Verifier)

// WithClientKeysPerItem keeps client keys on the host instead of registering them: SetClientKey and
// SetClientEd25519Key only record the key, and each request carries its client's key to the engine
// (sbv_mixed_verify_batch), which groups the keys that repeat inside a flush on the device. No table is built per
// client key and no flush rebuilds a registry when a client appears, so this suits client populations that come and go
// between reconfigurations. Consenter keys stay registered. Off by default.
func WithClientKeysPerItem() Option { return func(v *Verifier) { v.clientKeysPerItem = true } }

// WithKeyCache reserves, on every device, the engine's grouped-key cache (sbv_key_cache_reserve) for up to p256 / p384 /
// ed25519 client keys: the tables the engine builds for keys that repeat inside a flush are kept, so the next flushes of
// the same clients skip the build. It pays off with WithClientKeysPerItem, whose keys travel with every request. The cache
// fills once and is never evicted; each key costs 32 KiB (P-256), 118 KiB (P-384) or 47.8 KiB (Ed25519) of device memory
// per GPU. Verdicts are the same with or without it. Off by default.
func WithKeyCache(p256, p384, ed25519 int) Option {
	return func(v *Verifier) { v.keyCache, v.keyCacheEvicting = [3]int{p256, p384, ed25519}, false }
}

// WithEvictingKeyCache is WithKeyCache with a cache that replaces its least recently used tables when full
// (sbv_key_cache_reserve_evicting): for client populations larger than the cache, or that change over time. Each capacity
// is rounded up to a multiple of 16. Give it more ways than the clients that should stay resident, because keys hash into
// sets of 16 unevenly: 4,096 ways held all of 1,024 hot keys, and 1,024 ways held 921. Verdicts are the same with or
// without it. Off by default.
func WithEvictingKeyCache(p256, p384, ed25519 int) Option {
	return func(v *Verifier) { v.keyCache, v.keyCacheEvicting = [3]int{p256, p384, ed25519}, true }
}

// KeyCacheStats returns, for scheme 0 (P-256), 1 (P-384) or 2 (Ed25519), the capacity, resident tables, hits, misses,
// evictions and inserts given up of the grouped-key cache, summed over devices (sbv_key_cache_stats_ex).
func (v *Verifier) KeyCacheStats(scheme uint8) ([6]uint64, error) {
	var out [6]C.uint64_t
	if rc := C.sbv_key_cache_stats_ex(v.eng, C.uint8_t(scheme), &out[0]); rc != 0 {
		return [6]uint64{}, fmt.Errorf("sbv_key_cache_stats_ex failed: %d: %s", int(rc), C.GoString(C.sbv_last_error(v.eng)))
	}
	var r [6]uint64
	for i := range out {
		r[i] = uint64(out[i])
	}
	return r, nil
}

// Verifier implements api.Verifier.
type Verifier struct {
	eng *C.sbv_engine

	mu         sync.RWMutex
	verSeq     uint64
	registry   [][64]byte          // slot -> X||Y
	slots      map[[64]byte]uint32 // key -> slot
	consenters map[uint64]uint32
	clients    map[string]uint32
	edRegistry [][32]byte          // Ed25519 slot -> key, as the consenter or client registered it
	edSlots    map[[32]byte]uint32 // Ed25519 key -> slot
	edKeys     map[uint64]uint32   // consenters with crypto/ed25519 keys: their Ed25519 slot
	edClients  map[string]uint32   // clients with crypto/ed25519 keys: their Ed25519 slot
	dirty      bool                // the ECDSA registry differs from the engine's
	edDirty    bool                // the Ed25519 registry differs from the engine's

	clientKeysPerItem bool                 // WithClientKeysPerItem
	clientKeys        map[string]clientKey // client keys kept on the host (WithClientKeysPerItem)
	keyCache          [3]int               // WithKeyCache / WithEvictingKeyCache: tables per scheme
	keyCacheEvicting  bool                 // WithEvictingKeyCache

	pool sync.Pool // *pinned: one block of page-locked memory per in-flight batch

	agg *aggregator
}

// New opens the engine on the given CUDA devices (1, 2, 4 or 8 of one box).
func New(devices []int, opts ...Option) (*Verifier, error) {
	ords := make([]C.int, len(devices))
	for i, d := range devices {
		ords[i] = C.int(d)
	}
	var eng *C.sbv_engine
	if rc := C.sbv_create(&ords[0], C.int(len(devices)), &eng); rc != 0 {
		return nil, fmt.Errorf("sbv_create failed: %d (there is no CPU fallback)", int(rc))
	}
	v := &Verifier{eng: eng, slots: map[[64]byte]uint32{}, consenters: map[uint64]uint32{}, clients: map[string]uint32{},
		edSlots: map[[32]byte]uint32{}, edKeys: map[uint64]uint32{}, edClients: map[string]uint32{}, clientKeys: map[string]clientKey{}}
	for _, o := range opts {
		o(v)
	}
	if c := v.keyCache; c != [3]int{} {
		name := "sbv_key_cache_reserve"
		var rc C.int
		if v.keyCacheEvicting {
			name = "sbv_key_cache_reserve_evicting"
			rc = C.sbv_key_cache_reserve_evicting(eng, C.size_t(c[0]), C.size_t(c[1]), C.size_t(c[2]))
		} else {
			rc = C.sbv_key_cache_reserve(eng, C.size_t(c[0]), C.size_t(c[1]), C.size_t(c[2]))
		}
		if rc != 0 {
			err := fmt.Errorf("%s failed: %d: %s", name, int(rc), C.GoString(C.sbv_last_error(eng)))
			C.sbv_destroy(eng)
			return nil, err
		}
	}
	v.pool.New = func() interface{} { return &pinned{} }
	v.agg = newAggregator(v.engineBatch, 200*time.Microsecond, 65536)
	return v, nil
}

func (v *Verifier) Close() { v.agg.stop(); C.sbv_destroy(v.eng) }

// fault: an engine fault is never a verdict. The reference maps a Verifier error to "bad signature"
// (internal/bft/view.go:839-842) or to Complain+Sync (view.go:386-393); a CUDA error must fail-stop,
// as the reference itself panics on unrecoverable local errors (view.go:412-414).
func (v *Verifier) fault(what string, rc C.int) {
	panic(fmt.Sprintf("sbv: %s: engine fault %d: %s", what, int(rc), C.GoString(C.sbv_last_error(v.eng))))
}

func (v *Verifier) slotOf(xy [64]byte) uint32 { // v.mu held
	if s, ok := v.slots[xy]; ok {
		return s
	}
	s := uint32(len(v.registry))
	v.registry = append(v.registry, xy)
	v.slots[xy] = s
	v.dirty = true
	return s
}

func (v *Verifier) edSlotOf(pub [32]byte) uint32 { // v.mu held
	if s, ok := v.edSlots[pub]; ok {
		return s
	}
	s := uint32(len(v.edRegistry))
	v.edRegistry = append(v.edRegistry, pub)
	v.edSlots[pub] = s
	v.edDirty = true
	return s
}

// A consenter or client holds one key: setting a key of one type removes any key of the other type it held, so a
// signature is never checked under a key the configuration no longer gives it.
func (v *Verifier) SetConsenterKey(id uint64, xy [64]byte) {
	v.mu.Lock()
	v.consenters[id] = v.slotOf(xy)
	delete(v.edKeys, id)
	v.mu.Unlock()
}
func (v *Verifier) SetClientKey(c string, xy [64]byte) {
	v.mu.Lock()
	if v.clientKeysPerItem {
		v.clientKeys[c] = clientKey{key: xy}
	} else {
		v.clients[c] = v.slotOf(xy)
		delete(v.edClients, c)
	}
	v.mu.Unlock()
}
func (v *Verifier) SetVerificationSequence(s uint64) { v.mu.Lock(); v.verSeq = s; v.mu.Unlock() }

// SetConsenterEd25519Key: consenter `id` signs with crypto/ed25519 (an Ed25519 identity, as Fabric 3 allows next to
// ECDSA ones). Its signatures are 64 raw bytes R || S over the message itself (no prehash).
func (v *Verifier) SetConsenterEd25519Key(id uint64, pub [32]byte) {
	v.mu.Lock()
	v.edKeys[id] = v.edSlotOf(pub)
	delete(v.consenters, id)
	v.mu.Unlock()
}

// SetClientEd25519Key: client `c` signs its requests with crypto/ed25519; the signature field of its requests is the
// 64-byte R || S over the signed bytes of the request. The key is registered: a key the registry has not seen yet makes
// the next flush rebuild the Ed25519 registry (see ResetKeys for the cost). With WithClientKeysPerItem the key is
// only recorded and travels with the client's requests.
func (v *Verifier) SetClientEd25519Key(c string, pub [32]byte) {
	v.mu.Lock()
	if v.clientKeysPerItem {
		k := clientKey{ed: true}
		copy(k.key[:], pub[:])
		v.clientKeys[c] = k
	} else {
		v.edClients[c] = v.edSlotOf(pub)
		delete(v.clients, c)
	}
	v.mu.Unlock()
}

// ResetKeys drops every key, ECDSA and Ed25519, of consenters and clients. Keys change only with a reconfiguration, i.e. a new verification
// sequence (dependencies.go:65-66): the application calls ResetKeys, re-registers the new configuration's keys
// and bumps the sequence, so rotated keys do not pile up in HBM (264 KiB per P-256 key and 384 KiB per Ed25519 key,
// per GPU). Registered Ed25519 client keys (SetClientEd25519Key) cost 384 KiB per GPU each, and each new one makes the
// next flush rebuild every Ed25519 table (about 8 ms per thousand keys): a deployment whose clients, of either scheme,
// come and go between reconfigurations should open the Verifier WithClientKeysPerItem, so that client keys travel with
// the requests and repeated ones are grouped on the device instead.
func (v *Verifier) ResetKeys() {
	v.mu.Lock()
	v.registry, v.slots = nil, map[[64]byte]uint32{}
	v.consenters, v.clients = map[uint64]uint32{}, map[string]uint32{}
	v.edRegistry, v.edSlots = nil, map[[32]byte]uint32{}
	v.edKeys, v.edClients = map[uint64]uint32{}, map[string]uint32{}
	v.clientKeys = map[string]clientKey{}
	v.dirty, v.edDirty = true, true
	v.mu.Unlock()
}

// syncRegistry pushes the key registries that changed to the engine (sbv_set_keys builds one comb table per ECDSA
// key, sbv_ed25519_set_keys one fixed-base table per Ed25519 key).
func (v *Verifier) syncRegistry() {
	v.mu.Lock()
	defer v.mu.Unlock()
	if v.edDirty {
		var pub *C.uint8_t
		if len(v.edRegistry) > 0 {
			pub = (*C.uint8_t)(unsafe.Pointer(&v.edRegistry[0][0]))
		}
		if rc := C.sbv_ed25519_set_keys(v.eng, C.size_t(len(v.edRegistry)), pub); rc != 0 {
			v.fault("sbv_ed25519_set_keys", rc)
		}
		v.edDirty = false
	}
	if !v.dirty {
		return
	}
	n := len(v.registry)
	if n == 0 {
		if rc := C.sbv_set_keys(v.eng, C.uint64_t(v.verSeq), 0, nil, nil, nil); rc != 0 {
			v.fault("sbv_set_keys", rc)
		}
		v.dirty = false
		return
	}
	ids := make([]C.uint64_t, n)
	curve := make([]C.uint8_t, n)
	xy := make([]byte, 96*n)
	for i, k := range v.registry {
		ids[i] = C.uint64_t(i)
		copy(xy[96*i+16:], k[:32])
		copy(xy[96*i+48+16:], k[32:])
	}
	if rc := C.sbv_set_keys(v.eng, C.uint64_t(v.verSeq), C.size_t(n), &ids[0], &curve[0], (*C.uint8_t)(unsafe.Pointer(&xy[0]))); rc != 0 {
		v.fault("sbv_set_keys", rc)
	}
	v.dirty = false
}

// pinned is one block of page-locked host memory from the engine (sbv_host_alloc): C memory, so cgo may hand it
// to the engine freely, and the engine DMAs from it without a staging copy.
type pinned struct {
	p   unsafe.Pointer
	cap int
}

func (b *pinned) reserve(n int) []byte {
	if n > b.cap {
		if b.p != nil {
			C.sbv_host_free(b.p)
		}
		b.cap = n + n/2 + 4096
		b.p = C.sbv_host_alloc(C.size_t(b.cap))
		if b.p == nil {
			panic("sbv: sbv_host_alloc failed")
		}
	}
	return unsafe.Slice((*byte)(b.p), b.cap)[:n]
}

// engineBatch verifies an aggregated batch in at most two calls, whatever keys its items hold: the items with registered
// keys in one sbv_mixed_verify_registered call, the items that carry their key (WithClientKeysPerItem) in one
// sbv_mixed_verify_batch call. The engine splits each call's items by scheme on the GPU, hashes each message there
// (SHA-256 for ECDSA, SHA-512(R || A || M) for Ed25519) and verifies it; verdicts are put back in the items' order.
func (v *Verifier) engineBatch(items []item) []byte {
	v.syncRegistry()
	ok := make([]byte, len(items))
	var reg, keyed []int
	for i := range items {
		if items[i].keyed {
			keyed = append(keyed, i)
		} else {
			reg = append(reg, i)
		}
	}
	for _, idx := range [][]int{reg, keyed} {
		if len(idx) == 0 {
			continue
		}
		if len(idx) == len(items) {
			v.engineCall(items, idx, ok)
			break
		}
		part := make([]byte, len(idx))
		v.engineCall(items, idx, part)
		for j, i := range idx {
			ok[i] = part[j]
		}
	}
	return ok
}

// engineCall verifies items[idx[0]], items[idx[1]], ... (all registered or all keyed) in one engine call, verdict j into
// ok[j]. The items are marshalled once, straight into pinned memory (one block per in-flight call, pooled):
// rows (96n: P-256 r || s or Ed25519 R || S in bytes [0, 64)) | keys (96n: P-256 X || Y or the Ed25519 key in bytes
// [0, 64)) or slots (4n) | off (8(n+1)) | scheme (n) | msgs.
func (v *Verifier) engineCall(items []item, idx []int, ok []byte) {
	n := len(idx)
	keyed := items[idx[0]].keyed
	total := 0
	for _, i := range idx {
		total += len(items[i].msg)
	}
	oKey := 96 * n
	oOff := oKey + 4*n
	if keyed {
		oOff = oKey + 96*n
	}
	oOff = (oOff + 7) &^ 7
	oScheme := oOff + 8*(n+1)
	oMsgs := oScheme + n
	pb := v.pool.Get().(*pinned)
	defer v.pool.Put(pb)
	buf := pb.reserve(oMsgs + total + 16)
	pos := 0
	binary.LittleEndian.PutUint64(buf[oOff:], 0)
	for j, i := range idx {
		it := &items[i]
		row := buf[96*j : 96*j+96]
		if it.ed {
			copy(row, it.edSig[:])
			buf[oScheme+j] = byte(C.SBV_ED25519)
		} else {
			copy(row, it.r[:])
			copy(row[32:], it.s[:])
			buf[oScheme+j] = byte(C.SBV_P256)
		}
		if keyed {
			copy(buf[oKey+96*j:oKey+96*j+96], it.key[:])
		} else {
			binary.LittleEndian.PutUint32(buf[oKey+4*j:], it.slot)
		}
		copy(buf[oMsgs+pos:], it.msg)
		pos += len(it.msg)
		binary.LittleEndian.PutUint64(buf[oOff+8*(j+1):], uint64(pos))
	}
	base := uintptr(pb.p)
	at := func(o int) *C.uint8_t { return (*C.uint8_t)(unsafe.Pointer(base + uintptr(o))) }
	off := (*C.uint64_t)(unsafe.Pointer(base + uintptr(oOff)))
	out := (*C.uint8_t)(unsafe.Pointer(&ok[0]))
	if keyed {
		if rc := C.sbv_mixed_verify_batch(v.eng, C.size_t(n), at(oScheme), at(oMsgs), off, at(0), at(oKey), out); rc != 0 {
			v.fault("sbv_mixed_verify_batch", rc)
		}
		return
	}
	if rc := C.sbv_mixed_verify_registered(v.eng, C.size_t(n), at(oScheme), at(oMsgs), off, (*C.uint32_t)(unsafe.Pointer(base+uintptr(oKey))), at(0),
		out); rc != 0 {
		v.fault("sbv_mixed_verify_registered", rc)
	}
}

// parseDER: strict SEQUENCE{INTEGER r, INTEGER s} as crypto/ecdsa.VerifyASN1 (minimal, non-negative,
// no trailing bytes).
func parseDER(sig []byte) (r, s [32]byte, ok bool) {
	readInt := func(p []byte, out *[32]byte) ([]byte, bool) {
		if len(p) < 2 || p[0] != 0x02 {
			return nil, false
		}
		l := int(p[1])
		p = p[2:]
		if l&0x80 != 0 || l == 0 || len(p) < l || p[0]&0x80 != 0 || (l > 1 && p[0] == 0 && p[1]&0x80 == 0) {
			return nil, false
		}
		v := p[:l]
		if len(v) > 1 && v[0] == 0 {
			v = v[1:]
		}
		if len(v) > 32 {
			return nil, false
		}
		copy(out[32-len(v):], v)
		return p[l:], true
	}
	if len(sig) < 2 || sig[0] != 0x30 {
		return
	}
	var body []byte
	switch {
	case sig[1] < 0x80:
		body = sig[2:]
		if len(body) != int(sig[1]) {
			return
		}
	case sig[1] == 0x81 && len(sig) >= 3 && sig[2] >= 0x80:
		body = sig[3:]
		if len(body) != int(sig[2]) {
			return
		}
	default:
		return
	}
	rest, good := readInt(body, &r)
	if !good {
		return
	}
	rest, good = readInt(rest, &s)
	return r, s, good && len(rest) == 0
}

func (v *Verifier) consenterItem(sig types.Signature) (item, error) {
	v.mu.RLock()
	slot, known := v.consenters[sig.ID]
	edSlot, isEd := v.edKeys[sig.ID]
	v.mu.RUnlock()
	if isEd {
		if len(sig.Value) != 64 { // crypto/ed25519.Verify rejects any other length
			return item{}, fmt.Errorf("malformed signature from %d", sig.ID)
		}
		it := item{ed: true, slot: edSlot, msg: sig.Msg}
		copy(it.edSig[:], sig.Value)
		return it, nil
	}
	if !known {
		return item{}, fmt.Errorf("unknown consenter %d", sig.ID)
	}
	r, s, ok := parseDER(sig.Value)
	if !ok {
		return item{}, fmt.Errorf("malformed signature from %d", sig.ID)
	}
	return item{r: r, s: s, slot: slot, msg: sig.Msg}, nil
}

// VerifyConsenterSig — dependencies.go:60-62. Called from one goroutine per commit vote
// (view.go:537-541): concurrent calls coalesce in the aggregator.
func (v *Verifier) VerifyConsenterSig(sig types.Signature, prop types.Proposal) ([]byte, error) {
	want, _ := hex.DecodeString(prop.Digest()) // pkg/types/types.go:50-69
	if len(sig.Msg) < 32 || !bytes.Equal(sig.Msg[:32], want) {
		return nil, errors.New("signature does not bind the proposal")
	}
	it, err := v.consenterItem(sig)
	if err != nil {
		return nil, err
	}
	if !v.agg.submit(it) {
		return nil, fmt.Errorf("invalid signature from %d", sig.ID)
	}
	return v.AuxiliaryData(sig.Msg), nil
}

// VerifyConsenterSigBatch is what the restated batch call sites use (view.go:630-644,
// viewchanger.go:702-722): one engine call for the whole slice.
func (v *Verifier) VerifyConsenterSigBatch(sigs []types.Signature, prop types.Proposal) []error {
	want, _ := hex.DecodeString(prop.Digest())
	errs := make([]error, len(sigs))
	var items []item
	var where []int
	for i, sig := range sigs {
		if len(sig.Msg) < 32 || !bytes.Equal(sig.Msg[:32], want) {
			errs[i] = errors.New("signature does not bind the proposal")
			continue
		}
		it, err := v.consenterItem(sig)
		if err != nil {
			errs[i] = err
			continue
		}
		items = append(items, it)
		where = append(where, i)
	}
	if len(items) > 0 {
		ok := v.engineBatch(items)
		for k, i := range where {
			if ok[k] == 0 {
				errs[i] = fmt.Errorf("invalid signature from %d", sigs[i].ID)
			}
		}
	}
	return errs
}

// VerifySignature — dependencies.go:63-64 (viewchanger.go:598, 660, 983, 1022, 1076).
func (v *Verifier) VerifySignature(sig types.Signature) error {
	it, err := v.consenterItem(sig)
	if err != nil {
		return err
	}
	if !v.agg.submit(it) {
		return fmt.Errorf("invalid signature from %d", sig.ID)
	}
	return nil
}

// request := u16be siglen || sig (DER, or R || S for an Ed25519 client) || u32be clen || client || u32be ilen || id || payload
func (v *Verifier) requestItem(val []byte) (item, types.RequestInfo, error) {
	if len(val) < 2 {
		return item{}, types.RequestInfo{}, errors.New("malformed request")
	}
	sl := int(binary.BigEndian.Uint16(val))
	if len(val) < 2+sl+8 {
		return item{}, types.RequestInfo{}, errors.New("malformed request")
	}
	sig, signed := val[2:2+sl], val[2+sl:]
	p := signed
	read := func() (string, bool) {
		if len(p) < 4 {
			return "", false
		}
		l := int(binary.BigEndian.Uint32(p))
		if len(p) < 4+l {
			return "", false
		}
		s := string(p[4 : 4+l])
		p = p[4+l:]
		return s, true
	}
	client, ok1 := read()
	id, ok2 := read()
	if !ok1 || !ok2 {
		return item{}, types.RequestInfo{}, errors.New("malformed request")
	}
	v.mu.RLock()
	slot, known := v.clients[client]
	edSlot, isEd := v.edClients[client]
	ck, keyed := v.clientKeys[client]
	v.mu.RUnlock()
	info := types.RequestInfo{ClientID: client, ID: id}
	if keyed {
		it := item{keyed: true, ed: ck.ed, key: ck.key, msg: signed}
		if ck.ed {
			if len(sig) != 64 {
				return item{}, types.RequestInfo{}, errors.New("malformed request signature")
			}
			copy(it.edSig[:], sig)
			return it, info, nil
		}
		var ok bool
		if it.r, it.s, ok = parseDER(sig); !ok {
			return item{}, types.RequestInfo{}, errors.New("malformed request signature")
		}
		return it, info, nil
	}
	if isEd {
		if len(sig) != 64 { // crypto/ed25519.Verify rejects any other length
			return item{}, types.RequestInfo{}, errors.New("malformed request signature")
		}
		it := item{ed: true, slot: edSlot, msg: signed}
		copy(it.edSig[:], sig)
		return it, info, nil
	}
	if !known {
		return item{}, types.RequestInfo{}, fmt.Errorf("unknown client %s", client)
	}
	r, s, ok := parseDER(sig)
	if !ok {
		return item{}, types.RequestInfo{}, errors.New("malformed request signature")
	}
	return item{r: r, s: s, slot: slot, msg: signed}, info, nil
}

// VerifyRequest — dependencies.go:58-59 (controller.go:239, 742-745; requestpool.go:335-354).
func (v *Verifier) VerifyRequest(val []byte) (types.RequestInfo, error) {
	it, info, err := v.requestItem(val)
	if err != nil {
		return types.RequestInfo{}, err
	}
	if !v.agg.submit(it) {
		return types.RequestInfo{}, errors.New("bad request signature")
	}
	return info, nil
}

func splitRequests(payload []byte) ([][]byte, bool) {
	var out [][]byte
	for len(payload) > 0 {
		if len(payload) < 4 {
			return nil, false
		}
		l := int(binary.BigEndian.Uint32(payload))
		if len(payload) < 4+l {
			return nil, false
		}
		out = append(out, payload[4:4+l])
		payload = payload[4+l:]
	}
	return out, true
}

// VerifyProposal — dependencies.go:56-57 (view.go:555): every request of the batch in ONE engine call.
func (v *Verifier) VerifyProposal(prop types.Proposal) ([]types.RequestInfo, error) {
	reqs, ok := splitRequests(prop.Payload)
	if !ok {
		return nil, errors.New("malformed proposal payload")
	}
	if uint64(prop.VerificationSequence) != v.VerificationSequence() {
		return nil, errors.New("verification sequence mismatch")
	}
	items := make([]item, 0, len(reqs))
	infos := make([]types.RequestInfo, 0, len(reqs))
	for _, rq := range reqs {
		it, info, err := v.requestItem(rq)
		if err != nil {
			return nil, err
		}
		items = append(items, it)
		infos = append(infos, info)
	}
	if len(items) > 0 {
		for i, ok := range v.engineBatch(items) {
			if ok == 0 {
				return nil, fmt.Errorf("bad signature on request %s", infos[i].ID)
			}
		}
	}
	return infos, nil
}

func (v *Verifier) VerificationSequence() uint64 { v.mu.RLock(); defer v.mu.RUnlock(); return v.verSeq }

func (v *Verifier) RequestsFromProposal(prop types.Proposal) []types.RequestInfo {
	reqs, ok := splitRequests(prop.Payload)
	if !ok {
		return nil
	}
	var infos []types.RequestInfo
	for _, rq := range reqs {
		if _, info, err := v.requestItem(rq); err == nil {
			infos = append(infos, info)
		}
	}
	return infos
}

// AuxiliaryData — dependencies.go:69-70: Msg = digest(32) || aux.
func (v *Verifier) AuxiliaryData(msg []byte) []byte {
	if len(msg) < 32 {
		return nil
	}
	return append([]byte(nil), msg[32:]...)
}

// ---- aggregator: deadline-flush coalescing of concurrent single-signature calls ----

type batch struct {
	items    []item
	ok       []byte
	done     chan struct{}
	deadline time.Time
}

type aggregator struct {
	fn     func([]item) []byte
	window time.Duration
	max    int
	mu     sync.Mutex
	open   *batch
	quit   chan struct{}
}

func newAggregator(fn func([]item) []byte, window time.Duration, max int) *aggregator {
	a := &aggregator{fn: fn, window: window, max: max, open: &batch{done: make(chan struct{})}, quit: make(chan struct{})}
	go a.run()
	return a
}

// flushLocked closes the open batch and hands it to its own goroutine: the ticker goroutine and the caller that
// filled the batch never wait for the engine, so consecutive batches overlap on the engine's lanes.
func (a *aggregator) flushLocked() {
	b := a.open
	if len(b.items) == 0 {
		return
	}
	a.open = &batch{done: make(chan struct{})}
	go func() {
		b.ok = a.fn(b.items) // an engine fault panics here: never a verdict
		close(b.done)
	}()
}

// submit blocks until the batch the item joined has been verified (size cap or deadline, whichever is
// first — processCommits blocks the view goroutine until Q-1 valid votes exist, view.go:531, so a
// lone call must never wait for a batch to fill).
func (a *aggregator) submit(it item) bool {
	a.mu.Lock()
	b := a.open
	idx := len(b.items)
	b.items = append(b.items, it)
	if idx == 0 {
		b.deadline = time.Now().Add(a.window)
	}
	if len(b.items) >= a.max {
		a.flushLocked()
	}
	a.mu.Unlock()
	<-b.done
	return b.ok[idx] != 0
}

func (a *aggregator) run() {
	t := time.NewTicker(a.window / 4)
	defer t.Stop()
	for {
		select {
		case <-a.quit:
			return
		case now := <-t.C:
			a.mu.Lock()
			if len(a.open.items) > 0 && !now.Before(a.open.deadline) {
				a.flushLocked()
			}
			a.mu.Unlock()
		}
	}
}

func (a *aggregator) stop() { close(a.quit) }
