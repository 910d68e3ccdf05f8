/*
 * garecon.h — C ABI of the H100 batch reconcile-diff engine (libgarecon.so).
 *
 * Drop-in boundary for ONE path of h3poteto/aws-global-accelerator-controller: the
 * desired-vs-actual decision logic that the Go controller runs per work item behind
 *   pkg/reconcile/reconcile.go:22-26   (KeyToObjFunc / ProcessDeleteFunc / ProcessCreateOrUpdateFunc,
 *                                       ProcessNextWorkItem)
 * and that bottoms out in the decision functions of pkg/cloudprovider/aws
 * (global_accelerator.go:31-570, route53.go:18-130,216-238,335-395, load_balancer.go:32-93) and
 * pkg/cloudprovider/provider.go:8-17.
 *
 * The reference has no FFI (CGO_ENABLED="0", Makefile:27); these entry points are what a cgo shim
 * for that path would bind (see INTEGRATION.md).  Plain pointers and sizes only: no C++ / torch types.
 *
 * Data model
 * ----------
 * Everything is struct-of-arrays.  Strings never travel as pointers: a string is a `gar_str`
 * (40-bit byte offset | 24-bit length) into the byte slab of the table group it belongs to
 * (`gar_objects.slab` or `gar_actual.slab`).  One-to-many relations are CSR: `x_begin[i] .. x_begin[i+1]`
 * indexes the child table, every `*_begin` array has n+1 entries.  Child rows keep the order in which
 * the reference would see them (map-free lists in API/list order): that order is part of the contract
 * because the change set is ordered.
 *
 * Ownership: the caller owns every input buffer and may free it as soon as gar_snapshot_load returns
 * (cgo must not let C retain Go pointers); the engine owns a change set until gar_changeset_free.
 * Errors: every call returns GAR_OK or a negative gar_rc; gar_last_error gives the text.  The engine
 * never aborts and has no CPU fallback: without a usable sm_90 device every call fails.
 * Threading: calls on one engine are serialised by an internal mutex and may come from any OS thread.
 */
#ifndef GARECON_H
#define GARECON_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GAR_ABI_VERSION 1u

/* ---------------------------------------------------------------- strings */

typedef uint64_t gar_str; /* bits 0..39 byte offset into the slab, bits 40..63 length in bytes */
#define GAR_STR_OFF_BITS 40
#define GAR_STR(off, len) (((uint64_t)(len) << GAR_STR_OFF_BITS) | (uint64_t)(off))
#define GAR_STR_OFF(s) ((uint64_t)(s) & ((1ull << GAR_STR_OFF_BITS) - 1))
#define GAR_STR_LEN(s) ((uint32_t)((uint64_t)(s) >> GAR_STR_OFF_BITS))
#define GAR_NONE 0xFFFFFFFFu /* "no row" in op arguments */
#define GAR_PENDING 0xFFFFFFFEu /* op argument: the resource an EARLIER op of the same object creates (see "Self-observation") */

/* ---------------------------------------------------------------- return codes */

typedef enum {
  GAR_OK = 0,
  GAR_E_INVALID = -1,  /* bad argument / malformed table (offset out of slab, non-monotone CSR ...) */
  GAR_E_NO_DEVICE = -2,/* no CUDA device, or device is not sm_90 */
  GAR_E_CUDA = -3,     /* a CUDA call failed; text in gar_last_error */
  GAR_E_STATE = -4,    /* call order wrong (diff before load ...) */
  GAR_E_NOMEM = -5
} gar_rc;

/* ---------------------------------------------------------------- desired side: the informer cache */

/* obj_kind — which lister the row came from (globalaccelerator/controller.go:39,41) */
enum { GAR_KIND_SERVICE = 0, GAR_KIND_INGRESS = 1 };
/* obj_spec_type — corev1.ServiceType, Service rows only (globalaccelerator/service.go:19) */
enum { GAR_SVC_CLUSTERIP = 0, GAR_SVC_NODEPORT = 1, GAR_SVC_LOADBALANCER = 2, GAR_SVC_EXTERNALNAME = 3 };
/* obj_flags */
enum {
  GAR_OBJ_HAS_LB_CLASS = 1u << 0,      /* Service: spec.loadBalancerClass != nil (service.go:20) */
  GAR_OBJ_HAS_INGRESS_CLASS = 1u << 1  /* Ingress: spec.ingressClassName != nil; value in obj_ingress_class (ingress.go:20) */
};

typedef struct gar_objects {
  uint32_t n_objects;
  const uint8_t *obj_kind;          /* [n] GAR_KIND_* */
  const uint8_t *obj_spec_type;     /* [n] GAR_SVC_* (0 for Ingress rows) */
  const uint8_t *obj_flags;         /* [n] GAR_OBJ_* */
  const gar_str *obj_ns;            /* [n] metadata.namespace */
  const gar_str *obj_name;          /* [n] metadata.name */
  const gar_str *obj_ingress_class; /* [n] *spec.ingressClassName (only if GAR_OBJ_HAS_INGRESS_CLASS) */
  const uint32_t *obj_ann_begin;    /* [n+1] -> ann_*: metadata.annotations (keys unique per object) */
  const uint32_t *obj_lbi_begin;    /* [n+1] -> lbi_*: status.loadBalancer.ingress[] in order */
  const uint32_t *obj_port_begin;   /* [n+1] -> port_*: Service: spec.ports[] in order (global_accelerator.go:506);
                                       Ingress: defaultBackend.service.port.number (if defaultBackend and its
                                       .service are set) followed by every rules[].http.paths[].backend.service
                                       .port.number in order (global_accelerator.go:544-555; named ports are 0) */
  uint32_t n_ann;
  const gar_str *ann_key;           /* [n_ann] */
  const gar_str *ann_val;           /* [n_ann] */
  uint32_t n_lbi;
  const gar_str *lbi_hostname;      /* [n_lbi] status.loadBalancer.ingress[].hostname ("" when only .ip is set) */
  uint32_t n_ports;
  const int32_t *port_number;       /* [n_ports] */
  const gar_str *port_proto;        /* [n_ports] Service: spec.ports[].protocol as written ("TCP","UDP",...); Ingress: len 0 */
  const uint8_t *slab;
  uint64_t slab_len;
} gar_objects;

/* ---------------------------------------------------------------- actual side: listed AWS snapshots */

/* lb_state — elbv2types.LoadBalancerStateEnum (global_accelerator.go:125) */
enum { GAR_LB_ACTIVE = 0, GAR_LB_PROVISIONING = 1, GAR_LB_ACTIVE_IMPAIRED = 2, GAR_LB_FAILED = 3 };
/* lis_proto — gatypes.Protocol */
enum { GAR_PROTO_TCP = 0, GAR_PROTO_UDP = 1 };
/* rec_type — route53types.RRType; only A is distinguished by the path (route53.go:362) */
enum { GAR_RR_OTHER = 0, GAR_RR_A = 1, GAR_RR_TXT = 2, GAR_RR_CNAME = 3, GAR_RR_AAAA = 4 };

/* Only columns the decisions read are part of the ABI.  Identifiers the executor needs to CALL AWS with
   (accelerator / listener / endpoint-group ARNs, hosted-zone ids) stay on the Go side, addressed by the row
   indices the ops carry. */
typedef struct gar_actual {
  /* ELBv2 DescribeLoadBalancers, every region listed (load_balancer.go:13-30).  A lookup is by
     (region, name); with duplicates the first row wins, as `range res.LoadBalancers` does. */
  uint32_t n_lbs;
  const gar_str *lb_region;
  const gar_str *lb_name;
  const gar_str *lb_dns;
  const gar_str *lb_arn;
  const uint8_t *lb_state;
  /* Global Accelerator: ListAccelerators order (global_accelerator.go:624-641) */
  uint32_t n_accels;
  const gar_str *acc_name;
  const gar_str *acc_dns;
  const uint8_t *acc_enabled;
  const uint32_t *acc_tag_begin;   /* [n_accels+1] -> tag_*: ListTagsForResource order (:643-652) */
  const uint32_t *acc_lis_begin;   /* [n_accels+1] -> lis_*: ListListeners(accelerator) order (:789-803) */
  uint32_t n_tags;
  const gar_str *tag_key;
  const gar_str *tag_val;
  uint32_t n_listeners;
  const uint8_t *lis_proto;
  const uint32_t *lis_pr_begin;    /* [n_listeners+1] -> pr_from: Listener.PortRanges[] */
  const uint32_t *lis_eg_begin;    /* [n_listeners+1] -> eg_*: ListEndpointGroups(listener) order (:885-898) */
  uint32_t n_port_ranges;
  const int32_t *pr_from;          /* PortRange.FromPort — the only field the comparison reads (:460-462) */
  uint32_t n_egs;
  const uint32_t *eg_ep_begin;     /* [n_egs+1] -> ep_id: EndpointDescriptions[] */
  uint32_t n_endpoints;
  const gar_str *ep_id;            /* EndpointDescription.EndpointId (:496) */
  /* Route53: ListHostedZones order (route53.go:199-214); records in ListResourceRecordSets order (:317-333).
     A by-name zone lookup takes the first row whose name matches exactly (:349-353). */
  uint32_t n_zones;
  const gar_str *zone_name;        /* with trailing dot, as AWS returns it */
  const uint32_t *zone_rec_begin;  /* [n_zones+1] -> rec_* */
  uint32_t n_records;
  const gar_str *rec_name;         /* as AWS returns it: trailing dot, '*' escaped as \052 */
  const uint8_t *rec_type;         /* GAR_RR_* */
  const uint8_t *rec_has_alias;    /* AliasTarget != nil */
  const gar_str *rec_alias_dns;    /* AliasTarget.DNSName (only if rec_has_alias) */
  const uint32_t *rec_val_begin;   /* [n_records+1] -> val_value: ResourceRecords[] */
  uint32_t n_values;
  const gar_str *val_value;        /* ResourceRecord.Value (TXT values keep their double quotes) */
  const uint8_t *slab;
  uint64_t slab_len;
} gar_actual;

/* ---------------------------------------------------------------- engine configuration */

typedef struct gar_config {
  uint32_t abi_version;      /* GAR_ABI_VERSION */
  int32_t device;            /* CUDA device ordinal */
  const char *cluster_name;  /* --cluster-name (cmd/controller/controller.go:33); NUL-terminated, copied */
  uint32_t flags;            /* GAR_FLAG_* */
} gar_config;
#define GAR_FLAG_STAGE_TIMING 1u /* bracket every stage with CUDA events; read them with gar_last_stage_timings */
#define GAR_FLAG_REPREPARE 2u    /* rebuild the snapshot's digests and hash indexes on EVERY diff instead of once per load:
                                    for measuring the complete pipeline (bench.py "value", ncu captures) */
#define GAR_FLAG_NO_ORPHANS 4u   /* gar_diff leaves the two orphan sections empty: nothing is ever deleted on the strength of a key being
                                    ABSENT from the object table.  Deletes then come only from objects in the table (unmanaged / de-annotated)
                                    and from keys passed explicitly to gar_diff_keys as deleted (the reference's own rule: cleanup runs on an
                                    observed delete event, globalaccelerator/controller.go:113-173) */
#define GAR_FLAG_ALLOW_EMPTY_CACHE 8u /* see "Orphan sweep precondition" below */
/* Orphan sweep precondition.  The orphan sections of gar_diff stand for the delete events of every owner key that is tagged on an
   AWS resource of this cluster but has no object in the table: they are only right when the table is the COMPLETE, SYNCED informer
   cache of the whole cluster (HasSynced() true on both informers, no namespace-scoped cache, no failed or partial list, all slices
   present in sharded mode).  A caller that cannot guarantee that must set GAR_FLAG_NO_ORPHANS.  As a last line of defence gar_diff
   refuses (GAR_E_STATE) to emit orphan deletes when the object table is EMPTY while owned resources exist — the signature of an
   informer that has not synced — unless GAR_FLAG_ALLOW_EMPTY_CACHE says the empty cache is real (the last object was deleted). */

/* ---------------------------------------------------------------- output: the change set */

/* Per (controller, object) status word:  bits 0..7 gar_status, bits 8..15 gar_detail, bits 16..23 gar_event */
typedef enum {
  GAR_ST_IGNORED = 0,     /* object fails the controller's event filter (service.go:18-26, ingress.go:19-27) */
  GAR_ST_OK = 1,          /* Result{}, nil -> Forget (reconcile.go:87-89) */
  GAR_ST_SKIP_NO_LB = 2,  /* status.loadBalancer.ingress empty (service.go:59-62): Result{}, nil */
  GAR_ST_REQUEUE_30S = 3, /* LB not active (global_accelerator.go:125-128) -> AddAfter(30s) */
  GAR_ST_REQUEUE_60S = 4, /* accelerator-by-hostname count != 1 (route53.go:68-77) -> AddAfter(1m) */
  GAR_ST_ERR_RETRY = 5,   /* error, not NoRetry -> AddRateLimited (reconcile.go:75-77) */
  GAR_ST_ERR_NORETRY = 6, /* *NoRetryError -> dropped (reconcile.go:73-74); not produced by a snapshot diff */
  GAR_ST_PANIC = 7        /* DetectCloudProvider indexes parts[len-2] of a <2-label hostname (provider.go:9-10) */
} gar_status;

typedef enum {
  GAR_D_NONE = 0,
  GAR_D_NOT_ELB = 1,            /* load_balancer.go:42 */
  GAR_D_PARSE_INTERNAL_ALB = 2, /* load_balancer.go:64 */
  GAR_D_PARSE_PUBLIC_ALB = 3,   /* load_balancer.go:73 */
  GAR_D_PARSE_NLB = 4,          /* load_balancer.go:90 */
  GAR_D_LB_NOT_FOUND = 5,       /* load_balancer.go:29 (or the API's LoadBalancerNotFound) */
  GAR_D_LB_DNS_MISMATCH = 6,    /* global_accelerator.go:122-124 */
  GAR_D_TOO_MANY_LISTENERS = 7, /* global_accelerator.go:808-810 */
  GAR_D_TOO_MANY_EGS = 8,       /* global_accelerator.go:902-904 */
  GAR_D_NO_HOSTED_ZONE = 9,     /* route53.go:338-340 */
  GAR_D_ACCEL_MANY = 10,        /* route53.go:68-72 */
  GAR_D_ACCEL_NONE = 11         /* route53.go:73-77 */
} gar_detail;

enum {
  GAR_EV_CREATED = 1u << 0, /* GlobalAcceleratorCreated / Route53RecordCreated event (service.go:116-118, route53/service.go:101-103) */
  GAR_EV_DELETED = 1u << 1  /* GlobalAcceleratorDeleted / Route53RecordDeleted event (service.go:82, route53/service.go:67) */
};
#define GAR_STATUS(st, detail, ev) ((uint32_t)(st) | ((uint32_t)(detail) << 8) | ((uint32_t)(ev) << 16))
#define GAR_STATUS_CODE(w) ((w) & 0xFFu)
#define GAR_STATUS_DETAIL(w) (((w) >> 8) & 0xFFu)
#define GAR_STATUS_EVENT(w) (((w) >> 16) & 0xFFu)

/* Op codes.  Every op stands for a mutation the reference performs in-line.  Arguments are row indices
   into the input tables (GAR_NONE = absent).  `obj` is GAR_NONE for orphan ops.
     op                    sub            a0      a1               a2
     GA_CREATE_CHAIN       j              lb      NONE             NONE     global_accelerator.go:136-148,213-232
     GA_UPDATE_ACCEL       j              accel   lb               NONE     :291-296
     GA_CREATE_LISTENER    j              accel   NONE             NONE     :298-307
     GA_UPDATE_LISTENER    j              accel   listener         NONE     :313-321
     GA_CREATE_EG          j              accel   listener|NONE    lb       :322-331 (NONE: listener made by the preceding op)
     GA_UPDATE_EG          j              accel   eg               lb       :337-345
     GA_DELETE_CHAIN       0              accel   listener|NONE    eg|NONE  :254-288 (listener/eg only if exactly one exists)
     R53_CREATE            (j<<20)|k      zone    accel            NONE     route53.go:100-113 (TXT owner record, then A alias)
     R53_UPSERT_A          (j<<20)|k      zone    accel            record   route53.go:115-124
     R53_DELETE_RECORD     phase          zone    record           value    route53.go:132-165
   j = lbIngress index within the object, k = hostname index within the split route53-hostname annotation.
   Self-observation.  The reference mutates AWS between the iterations of its lbIngress / hostname loops and re-lists, so a later
   iteration of the SAME object sees what an earlier one did (ListGlobalAcceleratorByResource finds the accelerator created for
   lbIngress 0 and takes the update path for lbIngress 1, global_accelerator.go:133-157; updateEndpointGroup REPLACES the
   endpoint list, :987-1002; a hostname repeated in the route53 annotation finds the record just created, route53.go:92-124).
   The change set reproduces that against the frozen snapshot: from the second lbIngress that reaches the update/create stage
   on, an object's ops are what the reference would decide AFTER its own earlier ops — never a second GA_CREATE_CHAIN or a
   second R53_CREATE for the same name.  Such ops name resources that do not exist yet with GAR_PENDING:
     GA_UPDATE_ACCEL  a0 = PENDING          the accelerator of this object's earlier GA_CREATE_CHAIN
     GA_UPDATE_EG     a0 = PENDING | accel, a1 = PENDING   the endpoint group made by this object's earlier GA_CREATE_CHAIN /
                                                           GA_CREATE_LISTENER+GA_CREATE_EG / GA_CREATE_EG for that accelerator
     R53_UPSERT_A     a2 = PENDING          the A record of this object's earlier R53_CREATE for the same hostname string
   (User tags that overwrite the managed / owner / cluster tag with another value make an accelerator invisible to the list
   call once written: every later lbIngress then creates again, as the reference would.)
   R53_DELETE_RECORD: phase 0 = owned alias set (FindOwneredARecordSets), a2 = first value row of that zone
   whose value is the owner value and whose record has the alias set's name; phase 1 = owner metadata set
   (findOwneredMetadataRecordSets), a2 = the matching value row (one op per matching value, as the reference
   appends the set once per matching value). */
typedef enum {
  GAR_OP_GA_CREATE_CHAIN = 1,
  GAR_OP_GA_UPDATE_ACCEL = 2,
  GAR_OP_GA_CREATE_LISTENER = 3,
  GAR_OP_GA_UPDATE_LISTENER = 4,
  GAR_OP_GA_CREATE_EG = 5,
  GAR_OP_GA_UPDATE_EG = 6,
  GAR_OP_GA_DELETE_CHAIN = 7,
  GAR_OP_R53_CREATE = 8,
  GAR_OP_R53_UPSERT_A = 9,
  GAR_OP_R53_DELETE_RECORD = 10
} gar_opcode;

enum { GAR_CTRL_GA = 0, GAR_CTRL_R53 = 1 };

/* One op = 6 little-endian u32 words. */
typedef struct gar_op {
  uint32_t head; /* bits 0..7 gar_opcode, bits 8..15 GAR_CTRL_*, bits 16..23 GAR_KIND_* of obj (0 for orphans) */
  uint32_t obj;  /* object row, GAR_NONE for orphan ops */
  uint32_t sub;  /* see table above */
  uint32_t a0, a1, a2;
} gar_op;
#define GAR_OP_HEAD(op, ctrl, kind) ((uint32_t)(op) | ((uint32_t)(ctrl) << 8) | ((uint32_t)(kind) << 16))
#define GAR_R53_SUB(j, k) (((uint32_t)(j) << 20) | (uint32_t)(k))

/* Section order of `ops` (canonical; see DESIGN.md "Change-set order"):
     [0] GA ops of cached objects, by object row, then reference statement order
     [1] GA orphan deletes (owner tag of this cluster, no such object in the cache), by accelerator row
     [2] R53 ops of cached objects, by object row, then reference statement order
     [3] R53 orphan deletes, by (zone, phase, record row, value row) */
enum { GAR_SEC_GA_OBJ = 0, GAR_SEC_GA_ORPHAN = 1, GAR_SEC_R53_OBJ = 2, GAR_SEC_R53_ORPHAN = 3, GAR_N_SECTIONS = 4 };

/* Per-object derived desired state (what the create/update calls are fed; global_accelerator.go:214-225,503-557) */
enum {
  GAR_DV_PROTO_UDP = 1u << 0,      /* listenerForService protocol: last tcp/udp port wins (:503-515) */
  GAR_DV_IP_PRESERVE = 1u << 1,    /* client-ip-preservation annotation == "true" (:225) */
  GAR_DV_IPV4 = 1u << 2,           /* ip-address-type annotation in {"ipv4","IPV4"} (:686-695) */
  GAR_DV_PORTS_FROM_ANN = 1u << 3, /* Ingress carries alb.ingress.kubernetes.io/listen-ports: desired ports are
                                      dports[dport_begin[i]..], not port_number[] (:526-542) */
  GAR_DV_GA_ELIGIBLE = 1u << 4,    /* wasLoadBalancerService / wasALBIngress */
  GAR_DV_GA_MANAGED = 1u << 5,     /* hasManagedAnnotation (controller.go:250-253) */
  GAR_DV_R53_ELIGIBLE = 1u << 6,   /* route53 controller filter (route53/controller.go:87-148) */
  GAR_DV_R53_ANNOTATED = 1u << 7   /* hasHostnameAnnotation (route53/controller.go:243-246) */
};

/* gar_tok_code — result of DetectCloudProvider + GetLBNameFromHostname for one lbIngress hostname */
typedef enum {
  GAR_TOK_ALB_INTERNAL = 0,
  GAR_TOK_ALB_PUBLIC = 1,
  GAR_TOK_NLB = 2,
  GAR_TOK_NOT_AWS = 3,          /* DetectCloudProvider error -> `continue` (service.go:88-92) */
  GAR_TOK_PANIC = 4,            /* < 2 labels */
  GAR_TOK_ERR_NOT_ELB = 5,
  GAR_TOK_ERR_INTERNAL_ALB = 6,
  GAR_TOK_ERR_PUBLIC_ALB = 7,
  GAR_TOK_ERR_NLB = 8
} gar_tok_code;

typedef struct gar_changeset {
  uint32_t n_objects;
  const uint32_t *status_ga;   /* [n_objects] */
  const uint32_t *status_r53;  /* [n_objects] */
  const uint32_t *derived;     /* [n_objects] GAR_DV_* */
  uint64_t n_ops;
  const gar_op *ops;           /* [n_ops] */
  uint64_t section_begin[GAR_N_SECTIONS + 1];
  /* hostname tokeniser results, one per lbIngress row (name/region are refs into gar_objects.slab) */
  uint32_t n_lbi;
  const uint8_t *tok_code;     /* [n_lbi] gar_tok_code */
  const gar_str *tok_name;     /* [n_lbi] */
  const gar_str *tok_region;   /* [n_lbi] */
  /* desired port lists parsed from the listen-ports annotation (objects with GAR_DV_PORTS_FROM_ANN) */
  const uint32_t *dport_begin; /* [n_objects+1] */
  uint64_t n_dports;
  const int32_t *dports;       /* [n_dports] */
  /* sharded mode only (NULL otherwise): global object row of each local object row; ops then carry global rows */
  const uint32_t *obj_gid;     /* [n_objects] */
  /* timings of this diff, CUDA events on the engine's stream */
  float ms_h2d;                /* snapshot upload (measured at gar_snapshot_load) */
  float ms_kernels;            /* first kernel .. last kernel */
  float ms_d2h;                /* result download */
  uint32_t kernel_launches;    /* kernels launched by this diff */
  void *opaque;                /* engine-private; do not touch */
} gar_changeset;

typedef struct gar_engine gar_engine;

/* ---------------------------------------------------------------- entry points */

/* Create an engine bound to one CUDA device.  Fails with GAR_E_NO_DEVICE when there is no sm_90 GPU. */
int gar_engine_create(const gar_config *cfg, gar_engine **out);
void gar_engine_destroy(gar_engine *e);

/* Validate and copy a snapshot to the device (replaces any previous snapshot).
   Stands for: lister.List() on the two informers + the paginated AWS lists the per-object path issues
   (global_accelerator.go:624-652,789-813,885-907; route53.go:199-214,317-333; load_balancer.go:13-30). */
int gar_snapshot_load(gar_engine *e, const gar_objects *desired, const gar_actual *actual);

/* Same, for buffers that already live in device memory of the engine's device (all pointers in the two
   structs are device pointers, the structs themselves are host memory).  No copy is made: the caller keeps
   the buffers alive until the next load or gar_engine_destroy.  Table validation is skipped.
   What the kernels assume of the caller's buffers (gar_snapshot_load provides the same for its own copies):
     - each of the two slabs has 32 readable bytes behind slab + slab_len (their values do not matter): string compares
       and hashes load 8 bytes at a time and the staged row passes copy whole 16-byte lines, both reaching past a string's end;
     - each slab base is best 16-byte aligned: the staged row passes copy a block's strings to shared memory only from a
       16-byte aligned slab, otherwise they read every string from the slab directly (same results, slower).  The 8-byte
       loads are aligned down, so a base that is not 8-byte aligned also has up to 7 bytes before it read;
     - every column holds its n (begin arrays n + 1) elements at the alignment of its element type, and nothing more. */
int gar_snapshot_attach_device(gar_engine *e, const gar_objects *desired, const gar_actual *actual);

/* Compute the complete change set for both controllers against the loaded snapshot and copy it to host.
   Stands for: one processCreateOrUpdate / processDelete per key (globalaccelerator/service.go:28-126,
   ingress.go:29-130, route53/service.go:29-111, ingress.go:20-104) evaluated against the frozen snapshot. */
int gar_diff(gar_engine *e, gar_changeset *out);

/* Device-resident variant: runs the kernels only and leaves the result on the device.  Only the counts
   (n_ops, section_begin, n_dports) and timings of `out` are filled; array pointers are DEVICE pointers
   valid until the next diff/load on this engine. */
int gar_diff_device(gar_engine *e, gar_changeset *out);

/* Incremental mode (SURVEY.md §8 row f4): the decisions of a batch of work-queue keys against the loaded snapshot.
   `rows` are the object rows whose keys fired (informer add/update events, globalaccelerator/controller.go:91-111);
   `deleted_*` are keys that are no longer in the cache (delete events, :113-173): kind + "ns/name".
   Stands for: ProcessNextWorkItem once per key (pkg/reconcile/reconcile.go:26-42) -> processCreateOrUpdate for the
   rows, processDelete for the deleted keys.  The snapshot's digests and hash indexes are built on the first diff after
   a load and reused by every later gar_diff / gar_diff_keys until the next load.
   Result layout: n_objects = n_rows; status_ga[k], status_r53[k], derived[k] belong to rows[k]; object-section ops
   follow the order of `rows` and carry the real object row in `obj`; the orphan sections hold the cleanup ops of the
   deleted keys in the order given (per key: processDelete order, i.e. accelerators in list order / per zone alias
   sets then owner metadata sets); they carry obj = GAR_NONE.  tok_* and dports are not produced (n_lbi = 0,
   n_dports = 0). */
typedef struct gar_keyset {
  uint32_t n_rows;
  const uint32_t *rows;            /* [n_rows] object rows, each < n_objects */
  uint32_t n_deleted;
  const uint8_t *deleted_kind;     /* [n_deleted] GAR_KIND_* */
  const char *const *deleted_key;  /* [n_deleted] NUL-terminated "ns/name" */
} gar_keyset;
int gar_diff_keys(gar_engine *e, const gar_keyset *keys, gar_changeset *out);

/* Read set: the resident AWS rows that the decisions of a keyset read, so that a worker fed by deltas can re-describe exactly
   those rows (as gar_snapshot_apply_actual input) before it calls gar_diff_keys on the same keyset.  The reference re-lists AWS
   inside every reconcile; a resident snapshot only sees what the worker re-lists, and this call says what that must be.
   The units are gar_actual_delta's: an LB row, an accelerator with its whole subtree, a zone with its whole record list.
   Rules (a superset of what gar_diff_keys reads, independent of which branch each decision takes):
     - for each row i of keys->rows and each lbIngress j of i whose tokeniser code is GAR_TOK_ALB_INTERNAL, GAR_TOK_ALB_PUBLIC or
       GAR_TOK_NLB: the first LB row with that (region, name), or a miss entry when there is none; and the first two accelerators
       of this cluster (managed, cluster tag) whose target-hostname tag equals the lbIngress hostname (what the Route53 count
       gate reads);
     - for each row i: every accelerator of its owned-accelerator list (the list of the lowest row with i's key, as the decisions
       read it); the zone of every owner value of its key; and the zone GetHostedZone finds for every piece of
       strings.Split(route53-hostname annotation, ",") — a piece without a zone adds nothing (a new zone arrives through the
       worker's ListHostedZones comparison and gar_snapshot_apply_zones);
     - for each deleted key: the accelerators its cleanup deletes (owner tag of the key) and the zones of the owner values its
       Route53 cleanup finds.
   Guarantee: change any resident row outside the set, in any column that does not decide membership (LB region and name,
   accelerator tags, zone name, record values that are an owner value of a key in the set), apply it with
   gar_snapshot_apply_actual, and gar_diff_keys of the same keyset returns the identical change set (when a replaced subtree or
   record list changes its number of children, the listener, endpoint-group, record and value rows the ops name are renumbered
   by the new layout, nothing else).
   Limitation: a resource that becomes owned out of band (an accelerator whose tags are edited to name a key, a record given an
   owner value) is outside the set until it is listed; the periodic full re-list covers it.
   Validation is gar_diff_keys' (rows < n_objects, deleted keys a kind plus a NUL-terminated "ns/name"); GAR_E_INVALID changes
   nothing.  GAR_E_STATE before a load and on a sharded sub-snapshot (or once gar_shard_route has run on the loaded slice).  An
   attached snapshot is allowed.  The call prepares a stale snapshot exactly as gar_diff_keys would (the object side after an
   object delta or compaction, everything after an AWS or zone delta, ix_owner / ix_val when deleted keys need them); it changes
   nothing resident and leaves the recorded launch sequence as gar_diff_keys does: the next full diff replays if it would have.
   The arrays are engine-owned pinned host memory, valid until gar_read_set_free. */
typedef struct gar_readset {
  uint32_t n_lbs;
  const uint32_t *lb_rows;         /* [n_lbs] ascending, distinct resident LB rows */
  uint32_t n_lb_misses;            /* probes that found no LB row, ascending by (row, j), one per lbIngress: */
  const uint32_t *lb_miss_obj;     /*   [n_lb_misses] object row */
  const uint32_t *lb_miss_j;       /*   [n_lb_misses] lbIngress index within the object */
  const gar_str *lb_miss_name;     /*   [n_lb_misses] tokenised LB name, and */
  const gar_str *lb_miss_region;   /*   [n_lb_misses] region: refs into the resident object slab (gar_snapshot_read_slab) */
  uint32_t n_accels;
  const uint32_t *acc_rows;        /* [n_accels] ascending, distinct resident accelerator rows (whole subtrees) */
  uint32_t n_zones;
  const uint32_t *zone_rows;       /* [n_zones] ascending, distinct resident zone rows (whole record lists) */
  void *opaque;                    /* engine-private; do not touch */
} gar_readset;
int gar_read_set(gar_engine *e, const gar_keyset *keys, gar_readset *out);
void gar_read_set_free(gar_engine *e, gar_readset *rs);

/* ---------------------------------------------------------------- object deltas: keeping the resident snapshot current
   Informer events (add / update / delete of a Service or Ingress) applied to the loaded object table on the device, so that
   gar_diff_keys (and gar_diff, gar_bindings_diff) see them without a reload.  The AWS tables are left as loaded.
   A key is (kind, "ns/name").  Rules:
     - a key appears at most once per delta, counting deletes and upserts together (the caller coalesces events, as the
       workqueue does); otherwise GAR_E_INVALID;
     - deletes run first, in the given order: the key's row (the lowest row at that moment if several rows carry the key;
       a load may hold duplicates, an informer never does) is removed; unless it is the last row, the current last row moves
       into it (moved_from).  n_objects decreases by one.  A key that is not present is a no-op (deleted_row = GAR_NONE);
     - upserts run next, in the given order: a present key (lowest row) is replaced in place, an absent one appended as
       row n_objects.
   The table stays dense (object row order has no meaning: informer List order is unspecified), so every later call sees a
   table exactly like the one a gar_snapshot_load of the same objects would give, with two exceptions that the change set
   shows: tok_name / tok_region reference the resident object slab, where the strings of delta k sit at its slab_base.
   The resident object slab is append-only: strings of replaced and deleted rows stay until gar_snapshot_compact (below) drops
   them; slab_len tells the caller when a compaction is worth it.
   Atomic: the upsert table passes the checks of gar_snapshot_load (string references inside its own slab, monotone CSRs,
   kind / spec-type range, the ns/name layout rule) and the key rule above before anything resident changes; on
   GAR_E_INVALID the snapshot is unchanged.  A CUDA error in the middle leaves no loaded snapshot: later deltas return
   GAR_E_STATE and diffs fail until the next load.  GAR_E_STATE before any load, on an attached snapshot (gar_snapshot_attach_device), once gar_shard_route has run on
   the loaded slice, and on a sharded sub-snapshot.  The call drops the recorded launch sequence of the full diff.  The
   digests and indexes of the AWS tables stay prepared; the object side is rebuilt by the next diff. */
typedef struct gar_object_delta {
  const gar_objects *upserts;      /* added or updated objects: a complete table with its own slab, packed like a load's;
                                      NULL or n_objects == 0: no upserts */
  uint32_t n_deleted;
  const uint8_t *deleted_kind;     /* [n_deleted] GAR_KIND_* */
  const char *const *deleted_key;  /* [n_deleted] NUL-terminated "ns/name" (as in gar_keyset) */
} gar_object_delta;
typedef struct gar_delta_result {  /* arrays are caller-allocated */
  uint32_t *upsert_row;            /* [upserts->n_objects] final row of each upserted object */
  uint32_t *deleted_row;           /* [n_deleted] row the key had when it was removed; GAR_NONE if it was not in the cache */
  uint32_t *moved_from;            /* [n_deleted] row whose object moved into deleted_row[k]; GAR_NONE if none moved */
  uint32_t n_objects;              /* resident rows after the delta */
  uint64_t slab_base;              /* offset of this delta's upsert slab inside the resident object slab (16-byte aligned);
                                      0 when the delta has no upserts */
  uint64_t slab_len;               /* resident object slab bytes after the delta, strings of replaced rows included */
} gar_delta_result;
int gar_snapshot_apply_objects(gar_engine *e, const gar_object_delta *d, gar_delta_result *out);

/* ---------------------------------------------------------------- AWS deltas: re-listed AWS resources
   What a worker re-lists after executing ops (or after a requeue) applied to the loaded AWS tables on the device, so that the
   next batch diffs against what it just did instead of a stale list, without a reload.  The units are the list calls:
     load balancer   one DescribeLoadBalancers row                                        addressed by resident LB row
     accelerator     DescribeAccelerator + ListTagsForResource + ListListeners + ListEndpointGroups: the whole subtree
                     (tags, listeners, port ranges, endpoint groups, endpoints)          addressed by resident accelerator row
     hosted zone     ListResourceRecordSets(zone): the zone's complete record list        addressed by resident zone row
   (Hosted zones are added and removed by gar_snapshot_apply_zones, below.)  Rules:
     - order preserving: list order is part of the contract (the first (region, name) LB row wins, an owner's accelerators
       are visited in list order, the first matching alias in a zone wins).  Deleted LB and accelerator rows are removed and
       the survivors keep their relative order; a replaced row keeps its position; appended rows follow in delta order.  The
       new row of resident row r is r - #{deleted rows < r}; listeners, endpoint groups, records and values follow their
       parents exactly as a gar_snapshot_load of the resulting tables would lay them out, so the caller can compute every new
       row from its own data.  The result carries the table sizes as a cross-check;
     - a resident row appears at most once across the *_target and *_deleted arrays of its table, every row is < the table's
       size, zone_target entries are distinct, and delta zone k's zone_name equals resident zone zone_target[k]'s name byte
       for byte; otherwise GAR_E_INVALID;
     - the strings of `rows` are appended to the resident AWS slab at a 16-byte aligned slab_base (append-only, as for
       objects; slab_len tells the caller when a gar_snapshot_compact is worth it).
   Atomic: `rows` passes the checks gar_snapshot_load applies to an actual table (enums, monotone CSRs, strings inside its
   slab), and the rules above hold, before anything resident changes; on GAR_E_INVALID the snapshot is unchanged.  GAR_E_STATE
   in the same cases as gar_snapshot_apply_objects; after a CUDA error in the middle no snapshot is loaded.  Every later gar_diff,
   gar_diff_device, gar_diff_keys and gar_bindings_diff answers bit for bit as after a gar_snapshot_load of the same object table
   and the resulting AWS tables; object and AWS deltas may interleave freely.  The call drops the prepared state (digests,
   indexes) and the recorded launch sequence: the next diff prepares the snapshot as the first diff after a load does. */
typedef struct gar_actual_delta {
  const gar_actual *rows;          /* new rows: a complete actual table with its own slab, packed like a load's; NULL = none.  Its
                                      LBs and accelerators (with their subtrees) replace or append; its zone k carries the new
                                      record list of resident zone zone_target[k] and must have that zone's name */
  const uint32_t *lb_target;       /* [rows->n_lbs]    resident LB row replaced by delta row k, or GAR_NONE = append */
  const uint32_t *acc_target;      /* [rows->n_accels] the same for accelerators (the whole subtree is replaced) */
  const uint32_t *zone_target;     /* [rows->n_zones]  resident zone row whose record list is replaced */
  uint32_t n_lb_deleted;
  const uint32_t *lb_deleted;      /* [n_lb_deleted]  resident LB rows */
  uint32_t n_acc_deleted;
  const uint32_t *acc_deleted;     /* [n_acc_deleted] resident accelerator rows */
} gar_actual_delta;
typedef struct gar_actual_delta_result {
  uint32_t n_lbs, n_accels, n_tags, n_listeners, n_port_ranges, n_egs, n_endpoints, n_records, n_values; /* after the delta */
  uint64_t slab_base;              /* offset of this delta's slab inside the resident AWS slab (16-byte aligned); 0 when `rows`
                                      is NULL or holds no LB, accelerator or zone */
  uint64_t slab_len;               /* resident AWS slab bytes after the delta, strings of replaced rows included */
} gar_actual_delta_result;
int gar_snapshot_apply_actual(gar_engine *e, const gar_actual_delta *d, gar_actual_delta_result *out);

/* ---------------------------------------------------------------- zone deltas: hosted zones added and removed
   A changed ListHostedZones answer applied to the loaded zone table on the device, with the record sets of the zones it adds
   and removes, so that a CreateHostedZone or DeleteHostedZone needs no reload (and no re-list of everything else).  Zone order
   is part of the contract: the zone walk takes the first row whose name matches, a public and a private zone may share a name,
   and a new subzone changes the zone of every hostname below it.  Rules:
     - new order: for r = 0 .. n_zones (the resident count), first the new zones with added_at == r in delta order, then
       resident zone r unless it is deleted.  So surviving resident row r becomes
         r - #{deleted rows < r} + #{k : added_at[k] <= r},
       and new zone k gets row
         added_at[k] - #{deleted rows < added_at[k]} + k.
       Records and values follow their zones exactly as a gar_snapshot_load of the resulting tables would lay them out;
     - duplicate zone names are allowed (the first row wins, as after a load).  Zones cannot be renamed;
     - the strings of `added` are appended to the resident AWS slab at a 16-byte aligned slab_base, as for
       gar_snapshot_apply_actual; slab_base is 0 when nothing is added.  A later gar_snapshot_compact lays zone_name out in row
       order, as always.
   GAR_E_INVALID, with the snapshot unchanged: a deleted row >= n_zones or deleted twice; added_at[k] > n_zones or added_at
   decreasing; `added` holding load balancers, accelerators or any of their children; a NULL array with a non-zero count;
   anything gar_snapshot_load rejects in an actual table.  GAR_E_STATE in the cases of gar_snapshot_apply_actual (before a load,
   on an attached snapshot, once gar_shard_route has run on the loaded slice, on a sharded sub-snapshot).  After a CUDA error in
   the middle no snapshot is loaded.  Every later gar_diff, gar_diff_device, gar_diff_keys, gar_bindings_diff, object or AWS
   delta and compaction answers bit for bit as after a gar_snapshot_load of the same object table and the resulting AWS tables
   (tok_* reference the resident object slab, as after any delta).  The call drops the prepared state and the recorded launch
   sequence, as an AWS delta does. */
typedef struct gar_zone_delta {
  const gar_actual *added;      /* new hosted zones with their record lists, packed like a load's actual table with its own slab:
                                   n_zones, zone_name, zone_rec_begin, records, values.  Every other table is empty (n_lbs =
                                   n_accels = 0, CSRs {0}).  NULL or n_zones == 0: nothing added */
  const uint32_t *added_at;     /* [added->n_zones] resident zone row that new zone k is listed in front of; the resident n_zones =
                                   behind the last zone.  Non-decreasing in k */
  uint32_t n_deleted;
  const uint32_t *deleted;      /* [n_deleted] resident zone rows, removed together with their record sets; distinct */
} gar_zone_delta;
typedef struct gar_zone_delta_result {
  uint32_t n_zones, n_records, n_values;  /* after the delta */
  uint64_t slab_base, slab_len;           /* as in gar_actual_delta_result */
} gar_zone_delta_result;
int gar_snapshot_apply_zones(gar_engine *e, const gar_zone_delta *d, gar_zone_delta_result *out);

/* ---------------------------------------------------------------- record deltas: record sets edited inside resident zones
   Re-described record sets (ListResourceRecordSets with StartRecordName / StartRecordType / MaxItems) applied to the loaded record
   table on the device, so that a worker refreshes the record sets its keys read (gar_read_records, below) instead of whole zone
   record lists.  The scheme of the zone deltas, one level down.  Rules:
     - new order, inside every zone z: for each resident record r of z in order, first the delta records with rec_at == r in delta
       order, then r itself unless it is deleted; the delta records with rec_at == zone_rec_begin[z + 1] (behind z's last record)
       come last.  So resident record r becomes
         r - #{deleted rows < r} + #{k : rec_at[k] <= r},
       and delta record k becomes
         rec_at[k] - #{deleted rows < rec_at[k]} + k.
       An insert behind the last record of zone z and an insert in front of the first record of zone z + 1 share the rec_at value;
       the one of zone z comes first, which is delta order because zone_target ascends.  Replacing a record set is a delete of r
       plus an insert at r.  Values follow their records, and zone_rec_begin and everything else are laid out exactly as a
       gar_snapshot_load of the resulting tables would lay them out.  Load balancers, accelerators and zone rows do not move;
     - the strings of `rows` are appended to the resident AWS slab at a 16-byte aligned slab_base, as for gar_snapshot_apply_actual;
       slab_base is 0 when no record is inserted.
   GAR_E_INVALID, with the snapshot unchanged: anything gar_snapshot_load rejects in an actual table; `rows` holding load
   balancers, accelerators or any of their children; zone_target not strictly ascending or >= n_zones; a delta zone's zone_name
   different from its resident zone's; rec_at[k] outside [zone_rec_begin[z], zone_rec_begin[z + 1]] of its zone z (the next zone's
   interior included) or decreasing; a deleted row >= n_records or deleted twice; a NULL array with a non-zero count.  GAR_E_STATE
   in the cases of gar_snapshot_apply_actual (before a load, on an attached snapshot, once gar_shard_route has run on the loaded
   slice, on a sharded sub-snapshot); after a CUDA error in the middle no snapshot is loaded.  Every later gar_diff,
   gar_diff_device, gar_diff_keys, gar_bindings_diff, gar_read_set, gar_read_records, delta, compaction and export answers bit for
   bit as after a gar_snapshot_load of the same object table and the resulting AWS tables.  The call drops the prepared state and
   the recorded launch sequence, as an AWS delta does. */
typedef struct gar_record_delta {
  const gar_actual *rows;       /* record sets with their values, grouped by delta zone (zone_rec_begin), packed like a load's actual
                                   table with its own slab; n_lbs = n_accels = 0 and their CSRs {0}.  NULL / no records: inserts none */
  const uint32_t *zone_target;  /* [rows->n_zones] resident zone of delta zone k; strictly ascending; zone_name equal byte for byte */
  const uint32_t *rec_at;       /* [rows->n_records] resident record row that delta record k is listed in front of, inside
                                   [zone_rec_begin[z], zone_rec_begin[z + 1]] of its zone z (the end = behind the zone's last record);
                                   non-decreasing in k */
  uint32_t n_deleted;
  const uint32_t *deleted;      /* [n_deleted] resident record rows, removed with their values; distinct, < n_records */
} gar_record_delta;
typedef struct gar_record_delta_result {
  uint32_t n_records, n_values;  /* after the delta */
  uint64_t slab_base, slab_len;  /* as in gar_actual_delta_result */
} gar_record_delta_result;
int gar_snapshot_apply_records(gar_engine *e, const gar_record_delta *d, gar_record_delta_result *out);

/* Record read set: the resident record rows the Route53 decisions of a keyset read, the unit of gar_snapshot_apply_records.
   Rules (a superset of what gar_diff_keys reads, independent of which branch each decision takes):
     - for each row i of keys->rows: every owner value of i's owned-value list (the list of the lowest row with i's key, as the
       decisions read it; all zones): the record that carries it, and every alias record (rec_has_alias) of that zone whose name
       equals that record's name — FindOwneredARecordSets' result plus the sets its owner-value pass walks
       (route53.go:167-181,216-238);
     - for each deleted key: the same, for the owner values its cleanup finds through the owner-value index.
   Every row lies in a zone gar_read_set reports for the same keyset.
   Guarantee: insert, delete or change any record outside the set with gar_snapshot_apply_records, and gar_diff_keys of the same
   keyset returns the identical change set, except that the record and value rows the ops name are renumbered by the new layout.
   Limitation: a change that decides membership — a value that becomes an owner value of a key in the set, an alias record added
   under the name of a record in the set — is outside the set until it is listed, as for gar_read_set; the periodic full re-list
   covers it.
   Validation and GAR_E_STATE are gar_read_set's.  The call prepares a stale snapshot as gar_read_set does, changes nothing
   resident and leaves the recorded launch sequence as it was.  The array is engine-owned pinned host memory, valid until
   gar_read_records_free. */
typedef struct gar_record_readset {
  uint32_t n_records;
  const uint32_t *rec_rows;  /* [n_records] ascending, distinct resident record rows */
  void *opaque;              /* engine-private; do not touch */
} gar_record_readset;
int gar_read_records(gar_engine *e, const gar_keyset *keys, gar_record_readset *out);
void gar_read_records_free(gar_engine *e, gar_record_readset *rs);

/* ---------------------------------------------------------------- slab compaction: dropping the dead strings on the device
   Deltas only append to the two resident slabs.  gar_snapshot_compact rebuilds the slab of each selected group (`groups`: a
   mask of GAR_COMPACT_*) so that it holds exactly the strings the resident columns reference, entirely on the device: no byte
   comes from the host, and a worker that keeps its snapshot current by deltas needs neither a reload nor a host copy of the
   tables to get rid of the growth.
   Layout after the call (part of the contract: a caller can mirror it; deltas.compact / deltas.compact_actual of the Python
   package state it in numpy).  Per group, for each gar_str column in struct declaration order, the strings of rows 0 .. n-1
   back to back, no separators, no padding between strings or columns; slab_len is the sum of the live lengths.
     - objects: the key column comes first.  obj_ns[i] and obj_name[i] are slices of one "ns/name" string: the key is copied
       once, len(ns) + 1 + len(name) bytes from obj_ns[i]'s offset, and both references point into the copy (there is no
       separate name column).  Then obj_ingress_class, ann_key, ann_val, lbi_hostname, port_proto.
     - AWS: lb_region, lb_name, lb_dns, lb_arn, acc_name, acc_dns, tag_key, tag_val, ep_id, zone_name, rec_name, rec_alias_dns,
       val_value.
     - obj_ingress_class on a row without GAR_OBJ_HAS_INGRESS_CLASS, and rec_alias_dns on a row with rec_has_alias == 0, count as
       empty: whatever the reference held is not read (it may point outside the slab) and is replaced by an empty one.
     - an empty string keeps length 0 and gets the running offset of its column.
     - strings are never shared afterwards: two references to the same bytes become two copies (only the key pair stays
       shared).  For a hand-packed table that interned strings slab_len may therefore grow; `out` reports it, it is no error.
     - row order, every CSR and every fixed-width column are untouched.  The slab keeps GAR_SLAB_PAD zero bytes behind slab_len.
   Every later gar_diff, gar_diff_device, gar_diff_keys, gar_bindings_diff, gar_snapshot_apply_objects,
   gar_snapshot_apply_actual, gar_snapshot_apply_zones and gar_snapshot_apply_records answers bit for bit as before the call, except that tok_name / tok_region reference the new object
   slab (equal as the strings they name; gar_snapshot_read_slab resolves them) and later deltas report slab_base / slab_len
   relative to the compacted slab.
   groups == 0 or unknown bits: GAR_E_INVALID.  GAR_E_STATE in exactly the cases of gar_snapshot_apply_objects.  The new slabs and
   the rewritten reference columns are built in standby buffers and become resident together after the last kernel was queued: if
   a new slab cannot be allocated the call returns GAR_E_NOMEM and the snapshot is unchanged and usable (GAR_E_INVALID the same
   way if un-sharing would push a slab past 2^40 bytes); a CUDA error in the middle leaves no loaded snapshot, as for the deltas.
   The old slabs' memory is released.  Compacting the object group leaves the engine as an object delta does (the object side is
   rebuilt by the next diff, the AWS side stays prepared); compacting the AWS group drops the prepared state as an AWS delta
   does.  Both drop the recorded launch sequence. */
enum { GAR_COMPACT_OBJECTS = 1u << 0, GAR_COMPACT_ACTUAL = 1u << 1 };
typedef struct gar_compact_result {
  uint64_t obj_slab_before, obj_slab_len;   /* resident object slab bytes before / after (equal when not selected) */
  uint64_t act_slab_before, act_slab_len;   /* the same for the AWS slab */
} gar_compact_result;
int gar_snapshot_compact(gar_engine *e, uint32_t groups, gar_compact_result *out);

/* ---------------------------------------------------------------- export: the resident tables in host memory
   gar_snapshot_export copies the tables of each selected group (`groups`: a mask of GAR_COMPACT_*) into a host buffer of the
   caller, so that a snapshot kept current by deltas (the only up-to-date copy of the AWS side) can be checkpointed and later
   restored with one gar_snapshot_load instead of a re-list.
     - what is exported: the tables gar_snapshot_compact(groups) would leave resident at this moment: the same row order, CSRs
       and fixed-width columns, and the compaction layout above for the gar_str columns and the slab (the object key copied
       once, obj_ingress_class without its flag and rec_alias_dns without an alias empty, interned strings un-shared).  Right
       after a compaction the exported slab equals the resident one byte for byte.
     - buffer layout: the columns of the group in struct declaration order, each at a 16-byte aligned offset from the start of
       the buffer, the slab (slab_len bytes) last.  *obj_out / *act_out get the counts, slab_len and pointers into the buffer, so
       gar_snapshot_load(e2, obj_out, act_out) restores them directly; one exported group may be paired with a freshly packed
       table of the other (AWS tables from a checkpoint with a fresh informer list).
     - size query: obj_buf / act_buf == NULL for a selected group fills out->*_bytes / *_slab_len and writes nothing for that
       group.  The query runs the lengths pass and the scan of the export, so it costs device work.  A cap below the bytes
       needed returns GAR_E_INVALID with the needed bytes in `out`; nothing is written past the cap.
     - nothing resident changes: slabs, columns, the prepared state (digests, indexes, owned lists) and the recorded launch
       sequence stay as they were; the next diff replays if it would have replayed before.  The call only reads, so an attached
       snapshot can be exported too.
     - pinned host memory lets the copy overlap the gather on the device; pageable memory gives the same bytes, more slowly.
   GAR_E_INVALID: groups == 0 or unknown bits, a NULL *_out for a selected group, a buffer too small.  GAR_E_STATE before a load,
   on a sharded sub-snapshot and once gar_shard_route has run on the loaded slice.  GAR_E_NOMEM: device staging could not be
   allocated; the snapshot is unchanged.  A CUDA error returns GAR_E_CUDA and leaves the snapshot loaded, as a diff does. */
typedef struct gar_export_result {
  uint64_t obj_bytes, act_bytes;        /* buffer bytes the selected groups need (and, on success, used); 0 for a group not selected */
  uint64_t obj_slab_len, act_slab_len;  /* slab_len of the exported tables */
} gar_export_result;
int gar_snapshot_export(gar_engine *e, uint32_t groups, void *obj_buf, uint64_t obj_cap, gar_objects *obj_out, void *act_buf, uint64_t act_cap,
                        gar_actual *act_out, gar_export_result *out);

/* Copies `len` bytes at `off` of a resident slab to host memory (group = GAR_COMPACT_OBJECTS or GAR_COMPACT_ACTUAL, exactly one):
   how a caller reads the strings tok_name / tok_region name without mirroring the slab itself.  off + len beyond the resident
   slab_len, or a group that is not exactly one of the two: GAR_E_INVALID.  GAR_E_STATE before a load and on a sharded
   sub-snapshot (its strings live in the receive buffers). */
int gar_snapshot_read_slab(gar_engine *e, uint32_t group, uint64_t off, uint64_t len, void *dst);

/* ---------------------------------------------------------------- EndpointGroupBinding set-diff (SURVEY.md §8 row f3)
   The third controller's decisions (pkg/controller/endpointgroupbinding/reconcile.go:20-217): finalizer handling and the
   set difference between the load balancers of the referenced Service/Ingress and status.endpointIds.  Evaluated against
   the loaded snapshot (object cache, tokenised lbIngress hostnames, listed load balancers). */
enum { GAR_EGB_REF_NONE = 0, GAR_EGB_REF_SERVICE = 1, GAR_EGB_REF_INGRESS = 2 };
enum {
  GAR_EGB_DELETING = 1u << 0,       /* metadata.deletionTimestamp != nil (reconcile.go:27) */
  GAR_EGB_HAS_FINALIZERS = 1u << 1, /* len(metadata.finalizers) != 0 (:30) */
  GAR_EGB_OBSERVED = 1u << 2        /* status.observedGeneration == metadata.generation (:148) */
};
typedef struct gar_bindings {
  uint32_t n_bindings;
  const uint8_t *egb_flags;        /* GAR_EGB_* */
  const uint8_t *egb_ref_kind;     /* GAR_EGB_REF_*: spec.serviceRef / spec.ingressRef (:219-252) */
  const gar_str *egb_ref_key;      /* "<binding namespace>/<ref name>": the lister key of the referenced object */
  const gar_str *egb_eg_arn;       /* spec.endpointGroupArn */
  const uint32_t *egb_ep_begin;    /* [n_bindings+1] -> ep_id: status.endpointIds[] in order */
  uint32_t n_endpoint_ids;
  const gar_str *ep_id;
  uint32_t n_known_egs;            /* endpoint groups for which DescribeEndpointGroup succeeds (global_accelerator.go:867-876) */
  const gar_str *known_eg_arn;
  const uint8_t *slab;
  uint64_t slab_len;
} gar_bindings;

/* EGB ops (ctrl = GAR_CTRL_EGB, obj = binding row):
     EGB_ADD_FINALIZER      -            reconcileCreate  (:98-110)
     EGB_REMOVE_FINALIZER   -            reconcileDelete  (:36-47, :53-66)
     EGB_REMOVE_ENDPOINT    a0 = ep_id row                 RemoveLBFromEdnpointGroup (:80, :161)
     EGB_ADD_ENDPOINT       a0 = lb row                    AddLBToEndpointGroup (:172)
     EGB_UPDATE_WEIGHT      a0 = lb row                    UpdateEndpointWeight (:190)
     EGB_UPDATE_STATUS      -                              UpdateStatus (:87-90, :197-200)
   Go map iteration order (the `arns` map, :119,:139,:189) is unspecified; the canonical order here is first occurrence
   among the referenced object's lbIngress hostnames.  Statuses: GAR_ST_OK, GAR_ST_ERR_RETRY (GAR_D_*),
   GAR_ST_REQUEUE_30S (LB not active, global_accelerator.go:579-582), GAR_ST_REQUEUE_1S (:96), GAR_ST_PANIC (nil regional
   client when endpoints must be removed but the reference has no hostnames, :160; slice bounds in the delete loop, :84). */
enum { GAR_OP_EGB_ADD_FINALIZER = 11, GAR_OP_EGB_REMOVE_FINALIZER = 12, GAR_OP_EGB_REMOVE_ENDPOINT = 13, GAR_OP_EGB_ADD_ENDPOINT = 14,
       GAR_OP_EGB_UPDATE_WEIGHT = 15, GAR_OP_EGB_UPDATE_STATUS = 16 };
enum { GAR_CTRL_EGB = 2 };
enum { GAR_ST_REQUEUE_1S = 8 };
enum { GAR_D_REF_NOT_FOUND = 12, GAR_D_EG_NOT_FOUND = 13 };

/* Result: n_objects = n_bindings, status_ga[] holds the binding statuses, ops the EGB ops in binding order (one section);
   status_r53 / derived / tok_* / dports are not produced. */
int gar_bindings_diff(gar_engine *e, const gar_bindings *bindings, gar_changeset *out);

/* ---------------------------------------------------------------- sharded mode (SURVEY.md §8 row e, BASELINE configs[3])

   ONE cluster too large (or too slow) for one GPU, spread over n_ranks engines (one process per GPU).  Every rank loads
   (gar_snapshot_load) a SLICE: contiguous ranges of the object list and of each AWS list, in rank order (rank r holds
   global rows [base_r, base_r + n_r) of every table; nested rows travel with their parent), with these two rules:
     - the zone table (zone_name, zone_rec_begin) is complete and identical on every rank; a rank holds the record sets of
       whole zones only (other zones have empty record ranges), zone ranges ascending with the rank;
     - *_base give the global row of the slice's first row of each table.
   Both rules are checked on the device (a fingerprint of the zone table travels in the meta rows); a violation makes
   gar_shard_unpack return GAR_E_INVALID on the ranks that can see it — the host must propagate that to the other ranks
   before their next collective (shard.py does it with one all-reduce).
   Rows are then re-homed by key hash on the device in two exchanges the HOST performs between the calls below (the data
   path is torch.distributed all_to_all_single over NCCL in ranks.py, or any all-to-all):

     for round in 1, 2:
       gar_shard_route(e, &shard, round, meta, send_bytes)    meta[n_ranks][GAR_SHARD_META_WORDS]: row r describes the
                                                              blob for rank r; send_bytes[r] its size (multiple of 16)
       exchange the meta rows (all-to-all of GAR_SHARD_META_WORDS u64 per peer)
       gar_shard_pack(e, send)                                send: device buffer of sum(send_bytes), blobs back to back
       exchange the blobs (all-to-all, sizes from gar_shard_blob_bytes(received meta row))
       gar_shard_unpack(e, round, recv, recv_meta)            recv: the received blobs back to back, in rank order, with
                                                              32 readable bytes behind them (their values, like those of
                                                              the blobs' alignment gaps, do not matter).  The string bytes are NOT
                                                              copied: the sub-snapshot's strings live in BOTH rounds' receive
                                                              buffers, which must stay alive and unchanged until the last
                                                              diff of this exchange (the next gar_shard_route(.., 1) or
                                                              gar_snapshot_load ends their use; between that route call
                                                              and its second unpack gar_diff returns GAR_E_STATE)
   Round 1 moves every row to the shard its own key hashes to and one probe per lbIngress hostname to the "directory"
   shard of that hostname; round 2 returns the load balancer / by-hostname accelerators each probe resolves to.  After the
   second unpack the engine holds a self-contained sub-snapshot: gar_diff / gar_diff_device work as usual, n_objects is
   the number of objects homed here, obj_gid[] gives their global rows, ops carry GLOBAL rows and keep the canonical order
   within the shard (merge shards by (section, key row) for the cluster-wide order).  Stands for nothing in the reference
   (it has one process and no batch); semantics = gar_diff over the concatenated slices, which the tests check bit for bit. */
#define GAR_SHARD_MAX_RANKS 8
#define GAR_SHARD_META_WORDS 40
typedef struct gar_shard {
  uint32_t rank, n_ranks;
  uint32_t obj_base, lb_base, acc_base, lis_base, eg_base, rec_base, val_base;
} gar_shard;
int gar_shard_route(gar_engine *e, const gar_shard *shard, int round, uint64_t *meta, uint64_t *send_bytes);
int gar_shard_pack(gar_engine *e, void *send);
int gar_shard_unpack(gar_engine *e, int round, const void *recv, const uint64_t *recv_meta);
uint64_t gar_shard_blob_bytes(const uint64_t *meta_row);

/* Peer-memory exchange (one process per GPU on one NVLink / NVSwitch node): no collective on the data path.  Every rank maps the
   RECEIVE arenas of the other GPUs through CUDA IPC; gar_shard_pack_peers packs the rank's own blob in place and the others into a
   local stage from which a copy kernel on a high-priority stream pushes them into the peers' arenas over NVLink (16-byte coalesced
   stores), level group by level group while the later levels are still being packed (transfer and partitioning overlap).
   Alternatives kept behind environment switches for measurement: GAR_PEER_CE=1 (copy engines
   instead of the copy kernel), GAR_PEER_DIRECT=1 (the pack kernels store straight into the mapped arenas: 8-byte scattered
   stores over NVLink), GAR_PACK_TMA=1 (bulk stores from shared memory).  Per round:

     gar_shard_route(e, &shard, round, meta, send_bytes)
     all-gather the meta rows                                  -> all_meta[s][d] = row of source s for destination d
     gar_shard_arena(e, round, need, &ptr, handle, &cap)       need = sum over s of gar_shard_blob_bytes(all_meta[s][rank]);
                                                               (re)allocates this rank's arena of the round and exports it
     all-gather the handles; gar_shard_open_peers(e, round, handles)     (mappings are cached: re-opened only when a handle changed)
     gar_shard_pack_peers(e, round, all_meta)                  source s writes its blob for d at offset sum_{s' < s} blob bytes(s', d)
     barrier over the ranks (every pack has completed)         gar_shard_pack_peers has synchronised its own stream before returning
     gar_shard_unpack(e, round, ptr, column `rank` of all_meta)

   Same result as the send-buffer + all-to-all path above (tests compare both with the unsharded diff).  The host still moves
   the few hundred bytes of meta rows and handles (any all-gather); the bulk data never touches a collective library. */
#define GAR_SHARD_HANDLE_BYTES 96
int gar_shard_arena(gar_engine *e, int round, uint64_t need_bytes, void **arena, uint8_t *handle /* [GAR_SHARD_HANDLE_BYTES] */, uint64_t *capacity);
int gar_shard_open_peers(gar_engine *e, int round, const uint8_t *handles /* [n_ranks][GAR_SHARD_HANDLE_BYTES], rank order */);
int gar_shard_pack_peers(gar_engine *e, int round, const uint64_t *all_meta /* [n_ranks][n_ranks][GAR_SHARD_META_WORDS] */);

void gar_changeset_free(gar_engine *e, gar_changeset *cs);

const char *gar_last_error(const gar_engine *e); /* never NULL; valid until the next call on e */
const char *gar_version(void);

/* Bytes the diff must touch at least once: input slabs + fixed-width columns (each once)
   + 4 B per (controller, object) status + 24 B per op.  The roofline numerator (DESIGN.md §Measurement). */
uint64_t gar_algorithmic_bytes(const gar_engine *e, const gar_changeset *cs);

/* Per-stage device times of the last gar_diff / gar_diff_device (engine created with GAR_FLAG_STAGE_TIMING).
   Stages launched several times (index builds) are summed under one name.  Returns the number of stages. */
typedef struct gar_stage_timing {
  const char *name; /* static string */
  float ms;         /* CUDA-event time on the engine's stream */
  uint32_t launches;
  uint64_t bytes;   /* algorithmic bytes of the stage (DESIGN.md "Per-kernel byte model"), 0 if not modelled */
} gar_stage_timing;
uint32_t gar_last_stage_timings(gar_engine *e, gar_stage_timing *out, uint32_t cap);

/* Work counters of the last gar_diff / gar_diff_device / gar_diff_keys: exact sizes of the intermediate relations, for the
   per-kernel byte models of the roofline report (bench.py).  out[GAR_CTR_*]; returns the number of counters written. */
enum {
  GAR_CTR_R53_PAIRS = 0,   /* (object, route53 hostname) pairs evaluated by the r53_pairs stage (route53.go:84-124 loop bodies) */
  GAR_CTR_DPORTS = 1,      /* ports parsed from listen-ports annotations */
  GAR_CTR_LAUNCH_MODE = 2, /* how the last diff issued its launches: 0 eager, 1 recorded into a CUDA graph, 2 replayed from one.
                              Incremental and binding diffs always report 0 */
  GAR_CTR_N = 3
};
uint32_t gar_last_counters(gar_engine *e, uint64_t *out, uint32_t cap);

#ifdef __cplusplus
}
#endif
#endif /* GARECON_H */
